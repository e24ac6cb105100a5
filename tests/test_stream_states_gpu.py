"""Many streams' states saved and loaded in one call (lwb_streams_save / lwb_streams_load, Context.save_states /
load_states, sharding.migrate_streams), against the oracle.

Streams decode a first part of their packets, their states are saved, loaded into fresh streams of the same or a second
context, and both the loaded and the original streams decode the rest: the loaded streams' PCM must equal the oracle run
straight through and the uninterrupted streams' PCM, byte for byte, in every output format.  Only k_row_copy may run for
a save or a load.  The saved bytes are what lwb_stream_export_state gives, at any offset and buffer alignment; saves and
loads order with submits without a wait; a refused call changes nothing."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import lewton_b200 as L
from helpers import (ALL_KERNELS, RefStream, bits_equal, expect_kernels, launches_are_attributed, make_setup, mismatch_report,
                     random_floor1_y)
from lewton_b200 import _cabi as cabi

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPECTRUM, RESIDUE, HOST, DEVICE = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, cabi.MEM_DEVICE
F32P, I16P, F32I, I16I, F16P, F16I = (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED,
                                      cabi.OUT_F16_PLANAR, cabi.OUT_F16_INTERLEAVED)
FORMATS = [F32P, I16I, F16P, F32I, I16P, F16I]
DTYPE = {F32P: np.float32, F32I: np.float32, I16P: np.int16, I16I: np.int16, F16P: np.float16, F16I: np.float16}
PLANAR = {F32P, I16P, F16P}
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
# channels, blocksize_0, blocksize_1 (log2); ten channels take the four-kernel path
SETUPS = {"mono_256_2048": (1, 8, 11), "stereo_256_2048": (2, 8, 11), "stereo_512_4096": (2, 9, 12), "six_1024_1024": (6, 10, 10),
          "ten_256_2048": (10, 8, 11), "stereo_64_8192": (2, 6, 13)}
ROW_COPY_ONLY = dict(ran={"k_row_copy"}, not_ran=ALL_KERNELS - {"k_row_copy"})


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx2():
    c = L.Context(0)
    yield c
    c.close()


def mappings(C):
    return [{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}] if C == 2 else [{"coupling": [], "floor_of_channel": [0] * C}]


def setup_of(ctx, name):
    C, b0, b1 = SETUPS[name]
    return make_setup(ctx, C, b0, b1, modes=[(0, 0), (1, 0)], mappings=mappings(C), floors=[FLOOR])


def flags(bf):
    n = len(bf)
    prev, nxt = np.ones(n, np.uint8), np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


class Track:
    """One stream's packets (mode, prev, next, coefficients, floors) and the oracle's PCM for each, run straight through."""

    def __init__(self, oracle, rng, name, entry, n_packets, end_short=False, p_short=0.3):
        self.C, self.bs0, self.bs1 = SETUPS[name]
        bf = (rng.random(n_packets) >= p_short).astype(np.uint8)
        if end_short and n_packets:
            bf[-1] = 0
        prev, nxt = flags(bf)
        ref = RefStream(oracle, self.C, self.bs0, self.bs1, [(0, 0), (1, 0)], mappings(self.C), [FLOOR])
        self.packets, self.want = [], []
        for m, p, q in zip(bf, prev, nxt):
            n2 = 1 << ((self.bs1 if m else self.bs0) - 1)
            if entry == RESIDUE:
                x = (rng.standard_normal((self.C, n2)) * rng.integers(0, 2, (self.C, n2))).astype(np.float32)
                fl = [None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.25 else random_floor1_y(rng, FLOOR[0], len(FLOOR[1]))
                      for r in rng.random(self.C)]
                rc, o = ref.packet(int(m), int(p), int(q), x, fl)
            else:
                x = (rng.standard_normal((self.C, n2)) * 0.1).astype(np.float32)
                fl = None
                rc, o = ref.spectrum(int(m), int(p), int(q), x)
            assert rc == 0
            self.packets.append((int(m), int(p), int(q), x, fl))
            self.want.append(o)
        self.end_state = ref.pwr.data()

    def want_pcm(self, k0, k1):
        return np.concatenate([np.zeros((self.C, 0), np.float32)] + self.want[k0:k1], axis=1)


def decode(ctx, items, entry, fmt=F32P):
    """One host-memory batch: items = [(pwr, track, k0, k1)] decodes packets [k0, k1) of each track on pwr.  Returns the
    PCM of each chain as [C][n] in the format's dtype."""
    planar = fmt in PLANAR
    coeffs, kinds, ys, dense, chains = [], [], [], [], []
    coff = ooff = rows = 0
    for pwr, tr, k0, k1 in items:
        pk = tr.packets[k0:k1]
        n = sum(L.get_decoded_sample_count(pwr.setup, m, p, q) for m, p, q, _, _ in pk)
        chains.append(L.ChainSpec(pwr, [m for m, *_ in pk], [p for _, p, *_ in pk], [q for _, _, q, *_ in pk], coeff_offset=coff,
                                  packet_index=rows, out_offset=ooff, out_stride=n + 4 if planar else 0))
        for m, p, q, x, fl in pk:
            coeffs.append(x.ravel())
            coff += x.size
            if entry == RESIDUE:
                k, y, d = L.DecodedPacket(m, x, fl).pack()
                kinds.append(k)
                ys.append(y)
                dense.append(np.zeros_like(x) if d is None else d)
        rows += len(pk)
        ooff += tr.C * (n + 4) if planar else tr.C * n + 4
    kw = {}
    if entry == RESIDUE and kinds:
        kw = dict(floor_kind=np.concatenate(kinds), floor1_y=np.concatenate(ys), dense_floor=np.concatenate([d.ravel() for d in dense]))
    pcm = np.zeros(max(ooff, 1), DTYPE[fmt])
    coeffs = np.concatenate(coeffs) if coeffs else np.zeros(1, np.float32)
    L.decode_chains(ctx, chains, entry, HOST, coeffs, pcm, fmt, **kw)
    out = []
    for c, (pwr, tr, _, _) in zip(chains, items):
        assert c.status == 0 and c.packets_done == len(c.modes)
        n = c.n_samples
        if planar:
            out.append(np.stack([pcm[c.out_offset + k * c.out_stride: c.out_offset + k * c.out_stride + n] for k in range(tr.C)]))
        else:
            out.append(pcm[c.out_offset: c.out_offset + n * tr.C].reshape(n, tr.C).T.copy())
    return out


def as_format(x, fmt, oracle):
    if DTYPE[fmt] == np.int16:
        return oracle.quantise_i16(x)
    if DTYPE[fmt] == np.float16:
        return np.asarray(x, np.float32).astype(np.float16)
    return x


def same(a, b):
    if a.dtype == np.float32:
        return bits_equal(a, b)
    if a.dtype == np.float16:
        return a.shape == b.shape and bool(np.all((a.view(np.uint16) == b.view(np.uint16)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))))
    return a.shape == b.shape and np.array_equal(a, b)


class StateBuffer:
    """A state buffer of n floats: page-locked host memory or a device tensor, `shift` floats past a 16-byte boundary."""

    def __init__(self, ctx, memory, n, shift=0, fill=np.nan):
        self.memory = memory
        if memory == HOST:
            self.h = ctx.host_alloc(n + 4, np.float32)
            self.h[...] = fill
            self.arr = self.h[shift: shift + n]
            self.ptr = self.arr
        else:
            self.t = torch.full((n + 4,), float(fill), dtype=torch.float32, device="cuda:%d" % ctx.device)
            torch.cuda.synchronize()
            self.ptr = self.t.data_ptr() + 4 * shift
            self.shift = shift

    def read(self):
        return self.arr.copy() if self.memory == HOST else self.t.cpu().numpy()[self.shift: len(self.t) - 4 + self.shift]


CASES = [(name, memory, i) for i, (name, memory) in enumerate((n, m) for n in SETUPS for m in (HOST, DEVICE))]


@pytest.mark.parametrize("name,memory,i", CASES, ids=[f"{n}-{'host' if m == HOST else 'device'}" for n, m, _ in CASES])
def test_round_trip_against_oracle(ctx, ctx2, oracle, name, memory, i):
    """Decode part of every stream, save, load into fresh streams (this context or a second one), decode the rest: the
    loaded streams give the oracle's PCM and the uninterrupted streams' PCM, byte for byte."""
    rng = np.random.default_rng(1000 + i)
    entry = RESIDUE if i % 2 else SPECTRUM
    fmt = FORMATS[i % len(FORMATS)]
    dst_ctx = ctx2 if (i // 2) % 2 else ctx
    S, P2 = 6, 4
    P1 = [0, 1, 2, 3, 5, 7][:S]                    # short and long first parts; the first stream is saved empty
    tracks = [Track(oracle, rng, name, entry, p1 + P2, end_short=False) for p1 in P1]
    su, su_dst = setup_of(ctx, name), setup_of(dst_ctx, name)
    pwrs = [L.PreviousWindowRight(su) for _ in tracks]
    for got, tr, p1 in zip(decode(ctx, [(p, t, 0, p1) for p, t, p1 in zip(pwrs, tracks, P1)], entry), tracks, P1):
        assert bits_equal(got, tr.want_pcm(0, p1)), mismatch_report(got, tr.want_pcm(0, p1))
    offsets, total = L.state_offsets(pwrs)
    buf = StateBuffer(ctx, memory, total)
    with expect_kernels(ctx, **ROW_COPY_ONLY):
        slots, t = ctx.save_states(pwrs, buf.ptr, memory, offsets)
        t.wait()
    assert [(s.has, s.len) for s in slots] == [(not p.is_empty(), len(p)) for p in pwrs]
    fresh = [L.PreviousWindowRight(su_dst) for _ in tracks]
    with expect_kernels(dst_ctx, **ROW_COPY_ONLY):
        dst_ctx.load_states([L.StateSlot(f, s.offset, s.len, s.has) for f, s in zip(fresh, slots)], buf.ptr, memory).wait()
    for f, p in zip(fresh, pwrs):
        a, b = f.data(), p.data()
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b))
    loaded = decode(dst_ctx, [(f, t, p1, p1 + P2) for f, t, p1 in zip(fresh, tracks, P1)], entry, fmt)
    straight = decode(ctx, [(p, t, p1, p1 + P2) for p, t, p1 in zip(pwrs, tracks, P1)], entry, fmt)
    for got, ref, tr, p1 in zip(loaded, straight, tracks, P1):
        want = as_format(tr.want_pcm(p1, p1 + P2), fmt, oracle)
        assert same(got, ref), "loaded stream differs from the uninterrupted one"
        assert same(got, want), "loaded stream differs from the oracle"
    for f, tr in zip(fresh, tracks):
        assert bits_equal(f.data(), tr.end_state)


def odd_states(ctx, oracle, rng):
    """Streams in every kind of state: empty, has with len 0, short-block right halves (n0 / 2), long ones, and imported
    lengths that are not multiples of 4."""
    su = setup_of(ctx, "stereo_256_2048")
    pwrs = []
    pwrs.append(L.PreviousWindowRight(su))                                   # empty
    p = L.PreviousWindowRight(su)
    p.set_data(np.zeros((2, 0), np.float32))                                 # has = 1, len = 0
    pwrs.append(p)
    tr = Track(oracle, rng, "stereo_256_2048", SPECTRUM, 3, end_short=True)
    p = L.PreviousWindowRight(su)
    decode(ctx, [(p, tr, 0, 3)], SPECTRUM)
    assert len(p) == 128                                                      # n0 / 2
    pwrs.append(p)
    tr = Track(oracle, rng, "stereo_256_2048", SPECTRUM, 2)
    p = L.PreviousWindowRight(su)
    decode(ctx, [(p, tr, 0, 2)], SPECTRUM)
    pwrs.append(p)
    for n in (5, 1, 1023, 2):
        p = L.PreviousWindowRight(su)
        p.set_data(rng.standard_normal((2, n)).astype(np.float32))
        pwrs.append(p)
    return su, pwrs


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("shift,gap", [(0, 0), (1, 3), (3, 1)], ids=["aligned", "shift1-gap3", "shift3-gap1"])
def test_saved_values_equal_export_state(ctx, oracle, memory, shift, gap):
    """The saved rows are lwb_stream_export_state's, at offsets that are not multiples of 4 in an unaligned buffer; the
    gaps between slots keep what was there; loading them back gives the same states."""
    rng = np.random.default_rng(7 + shift)
    su, pwrs = odd_states(ctx, oracle, rng)
    offsets, off = [], gap
    for p in pwrs:
        offsets.append(off)
        off += 2 * len(p) + gap
    buf = StateBuffer(ctx, memory, off + gap, shift=shift, fill=-7.0)
    with expect_kernels(ctx, **ROW_COPY_ONLY):
        slots, t = ctx.save_states(pwrs, buf.ptr, memory, offsets)
        t.wait()
    got = buf.read()
    inside = np.zeros(got.size, bool)
    for p, s in zip(pwrs, slots):
        d = p.data()
        assert s.has == (d is not None) and s.len == (0 if d is None else d.shape[1])
        if d is not None:
            assert bits_equal(got[s.offset: s.offset + d.size].reshape(d.shape), d)
            inside[s.offset: s.offset + d.size] = True
    assert np.all(got[~inside] == -7.0), "a save wrote outside its slots"
    fresh = [L.PreviousWindowRight(su) for _ in pwrs]
    for f in fresh:
        f.set_data(np.ones((2, 64), np.float32))
    with expect_kernels(ctx, **ROW_COPY_ONLY):
        ctx.load_states([L.StateSlot(f, s.offset, s.len, s.has) for f, s in zip(fresh, slots)], buf.ptr, memory).wait()
    for f, p in zip(fresh, pwrs):
        assert f.is_empty() == p.is_empty() and len(f) == len(p)
        a, b = f.data(), p.data()
        assert a is None or bits_equal(a, b)


def submit(ctx, items, entry=SPECTRUM):
    """A host-memory submit of items [(pwr, track, k0, k1)] on page-locked arrays; returns (ticket, read) where read()
    gives each chain's f32 planar PCM once the ticket is done."""
    chains, coeffs, ooff, coff = [], [], 0, 0
    for pwr, tr, k0, k1 in items:
        pk = tr.packets[k0:k1]
        n = sum(L.get_decoded_sample_count(pwr.setup, m, p, q) for m, p, q, _, _ in pk)
        chains.append(L.ChainSpec(pwr, [m for m, *_ in pk], [p for _, p, *_ in pk], [q for _, _, q, *_ in pk], coeff_offset=coff,
                                  out_offset=ooff, out_stride=n))
        for *_, x, _ in pk:
            coeffs.append(x.ravel())
            coff += x.size
        ooff += tr.C * n
    cf = ctx.host_alloc(max(coff, 1), np.float32)
    cf[:coff] = np.concatenate(coeffs)
    pcm = ctx.host_alloc(max(ooff, 1), np.float32)
    t = ctx.submit_chains(chains, entry, HOST, cf, pcm, F32P)

    def read():
        t.wait()
        return [np.stack([pcm[c.out_offset + k * c.out_stride: c.out_offset + k * c.out_stride + c.n_samples] for k in range(tr.C)])
                for c, (_, tr, _, _) in zip(chains, items)]
    return t, read


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
def test_ordering_without_synchronising(ctx, oracle, memory):
    """submit, save, submit, load (back to the checkpoint), submit, with no wait in between: the third submit decodes
    from the checkpoint, so it repeats the second's PCM, and every PCM is the oracle's."""
    rng = np.random.default_rng(21)
    name = "stereo_256_2048"
    tracks = [Track(oracle, rng, name, SPECTRUM, 6) for _ in range(5)]
    su = setup_of(ctx, name)
    pwrs = [L.PreviousWindowRight(su) for _ in tracks]
    _, total = L.state_offsets(pwrs, lengths=[1024] * len(pwrs))
    buf = StateBuffer(ctx, memory, total)
    offsets = L.state_offsets(pwrs, lengths=[1024] * len(pwrs))[0]
    _, r1 = submit(ctx, [(p, t, 0, 3) for p, t in zip(pwrs, tracks)])
    slots, ts = ctx.save_states(pwrs, buf.ptr, memory, offsets)
    _, r2 = submit(ctx, [(p, t, 3, 6) for p, t in zip(pwrs, tracks)])
    tl = ctx.load_states([L.StateSlot(p, s.offset, s.len, s.has) for p, s in zip(pwrs, slots)], buf.ptr, memory)
    _, r3 = submit(ctx, [(p, t, 3, 6) for p, t in zip(pwrs, tracks)])
    assert ts.id < tl.id
    for a, b, c, tr in zip(r1(), r2(), r3(), tracks):
        assert bits_equal(a, tr.want_pcm(0, 3)) and bits_equal(b, tr.want_pcm(3, 6))
        assert np.array_equal(b.view(np.uint32), c.view(np.uint32))
    for p, tr in zip(pwrs, tracks):
        assert bits_equal(p.data(), tr.end_state)


def test_prepared_batch_replans_after_a_load(ctx, oracle):
    """A prepared batch executed after a load that changes its streams' state shape plans again and gives the oracle's
    PCM: here the load puts back the empty states the batch first ran from."""
    rng = np.random.default_rng(5)
    name = "stereo_256_2048"
    tr_list = [Track(oracle, rng, name, SPECTRUM, 2, p_short=0) for _ in range(3)]
    su = setup_of(ctx, name)
    pwrs = [L.PreviousWindowRight(su) for _ in tr_list]
    buf = StateBuffer(ctx, DEVICE, 4)
    slots, t = ctx.save_states(pwrs, buf.ptr, DEVICE, [0] * len(pwrs))     # all empty: nothing is written
    t.wait()
    assert all(not s.has and s.len == 0 for s in slots)
    # the same two packets per stream, step after step, on device memory (a captured plan)
    chains, coeffs, off, ooff = [], [], 0, 0
    for p, tr in zip(pwrs, tr_list):
        chains.append(L.ChainSpec(p, [m for m, *_ in tr.packets], [q for _, q, *_ in tr.packets], [q for _, _, q, *_ in tr.packets],
                                  coeff_offset=off, out_offset=ooff, out_stride=2048))
        for *_, x, _ in tr.packets:
            coeffs.append(x.ravel())
            off += x.size
        ooff += 2 * 2048
    d_coeffs = torch.from_numpy(np.concatenate(coeffs)).cuda()
    d_pcm = torch.zeros(ooff, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    b = L.Batch(ctx, chains, SPECTRUM, DEVICE, d_coeffs.data_ptr(), d_pcm.data_ptr(), F32P)

    def step():
        b.run()
        ctx.synchronize()
        b.collect()
        pcm = d_pcm.cpu().numpy()
        return [pcm[c.out_offset: c.out_offset + 2 * 2048].reshape(2, 2048)[:, :c.n_samples].copy() for c in chains]
    first = step()
    step()
    ctx.load_states(slots, buf.ptr, DEVICE)
    again = step()
    for a, c, tr in zip(first, again, tr_list):
        assert bits_equal(a, tr.want_pcm(0, 2)) and bits_equal(c, tr.want_pcm(0, 2))


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
def test_recovery_from_a_checkpoint(ctx, oracle, memory):
    """Save, run two steps, load the checkpoint, run the two steps again: byte-identical output."""
    rng = np.random.default_rng(33)
    tracks = [Track(oracle, rng, n, RESIDUE, 6) for n in ("stereo_256_2048", "stereo_256_2048", "stereo_256_2048")]
    su = setup_of(ctx, "stereo_256_2048")
    pwrs = [L.PreviousWindowRight(su) for _ in tracks]
    decode(ctx, [(p, t, 0, 2) for p, t in zip(pwrs, tracks)], RESIDUE)
    offsets, total = L.state_offsets(pwrs)
    buf = StateBuffer(ctx, memory, total)
    slots, _ = ctx.save_states(pwrs, buf.ptr, memory, offsets)
    run1 = [decode(ctx, [(p, t, k, k + 2) for p, t in zip(pwrs, tracks)], RESIDUE, I16I) for k in (2, 4)]
    ctx.load_states(slots, buf.ptr, memory)
    run2 = [decode(ctx, [(p, t, k, k + 2) for p, t in zip(pwrs, tracks)], RESIDUE, I16I) for k in (2, 4)]
    for s1, s2 in zip(run1, run2):
        for a, b in zip(s1, s2):
            assert np.array_equal(a, b)
    for k, step in zip((2, 4), run1):
        for a, tr in zip(step, tracks):
            assert np.array_equal(a, oracle.quantise_i16(tr.want_pcm(k, k + 2)))


def raw_call(fn, ctx, slots, memory, buf, ticket=True):
    arr = (cabi.StateSlot * max(len(slots), 1))()
    for a, (h, off, n, has) in zip(arr, slots):
        a.stream, a.offset, a.len, a.has = h, off, n, has
    t = C.c_uint64(0)
    rc = fn(ctx._h, arr, len(slots), memory, L.api._addr(buf), C.byref(t) if ticket else None)
    return rc, t.value, arr


def test_refusals_change_nothing(ctx, ctx2, oracle):
    """Every refused save or load returns its code with every stream state, (has, len), the buffer and the ticket
    sequence as they were."""
    rng = np.random.default_rng(3)
    su, su2 = setup_of(ctx, "stereo_256_2048"), setup_of(ctx2, "stereo_256_2048")
    tr = Track(oracle, rng, "stereo_256_2048", SPECTRUM, 2)
    a, b = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
    decode(ctx, [(a, tr, 0, 2)], SPECTRUM)
    b.set_data(np.full((2, 8), 3.0, np.float32))
    other = L.PreviousWindowRight(su2)
    dev = StateBuffer(ctx, DEVICE, 4096, fill=5.0)
    pinned = StateBuffer(ctx, HOST, 4096, fill=5.0)
    pageable = np.full(4096, 5.0, np.float32)
    lib = cabi.lib()
    save, load = lib.lwb_streams_save, lib.lwb_streams_load
    A, B, O = a._h, b._h, other._h
    refused = [
        (save, [(A, 0, 0, 0), (O, 2048, 0, 0)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),       # a stream of another context
        (load, [(A, 0, 8, 1), (O, 16, 8, 1)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),
        (save, [(A, 0, 0, 0), (A, 2048, 0, 0)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),       # a stream in two slots
        (load, [(B, 0, 8, 1), (B, 16, 8, 1)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),
        (load, [(A, 0, 8, 1), (B, 16, 5, 0)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),         # has == 0, len != 0
        (load, [(None, 0, 8, 1)], DEVICE, dev.ptr, True, cabi.ERR_INVALID),                     # no stream
        (save, [(A, 0, 0, 0)], 7, dev.ptr, True, cabi.ERR_INVALID),                             # bad memory space
        (save, [(A, 0, 0, 0)], DEVICE, None, True, cabi.ERR_INVALID),                           # NULL buffer
        (load, [(A, 0, 8, 1)], DEVICE, dev.ptr, False, cabi.ERR_INVALID),                       # NULL ticket
        (save, [(A, 0, 0, 0)], HOST, pageable.ctypes.data, True, cabi.ERR_INVALID),             # pageable host memory
        (load, [(A, 0, 8, 1)], HOST, pageable.ctypes.data, True, cabi.ERR_INVALID),
        (load, [(B, 0, 8, 1), (A, 16, 1025, 1)], DEVICE, dev.ptr, True, cabi.ERR_BUFFER),       # len > blocksize_1 / 2
        (save, [(B, 0, 0, 0), (A, (1 << 62) - 64, 0, 0)], DEVICE, dev.ptr, True, cabi.ERR_BUFFER),  # a range that wraps
        (load, [(A, 0, 8, 1), (B, (1 << 64) - 8, 8, 1)], HOST, pinned.ptr, True, cabi.ERR_BUFFER),
    ]
    before = [(p.is_empty(), len(p), p.data()) for p in (a, b, other)]
    _, t0 = ctx.save_states([], dev.ptr, DEVICE)
    for k, (fn, slots, memory, buf, with_ticket, code) in enumerate(refused):
        rc, t, arr = raw_call(fn, ctx, slots, memory, buf, with_ticket)
        assert rc == code, (k, rc, lib.lwb_last_error(ctx._h))
        assert t == 0, k
        assert all(x.len == s[2] and x.has == s[3] for x, s in zip(arr, slots)), k
    for p, (e, n, d) in zip((a, b, other), before):
        assert p.is_empty() == e and len(p) == n
        assert d is None or bits_equal(p.data(), d)
    assert np.all(dev.read() == 5.0) and np.all(pinned.read() == 5.0) and np.all(pageable == 5.0)
    _, t1 = ctx.save_states([], dev.ptr, DEVICE)
    assert t1.id == t0.id + 1, "a refused call issued a ticket"


def torchrun(args, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join("tests", "state_rank_worker.py"), *args]
    return subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)


def test_migrate_streams_two_ranks_one_gpu_gloo():
    """migrate_streams over gloo between two ranks that share one GPU (each its own context): half the streams move
    mid-decode through page-locked host memory, and the combined PCM is the oracle's."""
    r = torchrun(["gloo"], 29631)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "MIGRATE_OK gloo" in r.stdout


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_migrate_streams_two_gpus_nccl():
    """migrate_streams over NCCL between two GPUs: the states cross in device memory."""
    r = torchrun(["nccl"], 29632)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "MIGRATE_OK nccl" in r.stdout
