"""Chains at element offsets past 2^31 and 2^32, on every batch path, against the same batch at small offsets.

The ABI takes coeff_offset, packet_index, out_offset and out_stride as uint64_t.  A decode server with a 16 GiB f32 arena
writes at element 2^32, and one long 7.1 chain written interleaved passes element 2^31; an offset truncated to 32 bits
anywhere -- a host planner, a run descriptor, a kernel's index arithmetic -- would address some other part of the arena.
Each case here decodes one batch twice: once in ordinary arenas at small offsets, once with its coefficient, PCM and
packet-row offsets moved past 2^30, 2^31 or 2^32 (or across 2^32 inside a run, or with planes 2^32 + 4 elements apart) in
sparse arenas (sparse_arena.py) whose 32-bit images are mapped and sentinel-filled as well.  Packer bitstreams add the VQ
entry with run and entry offsets past 2^31 and 2^32, and floor-0 records at packet rows past 2^30.  Then:
- every chain matches the oracle (f32 bit for bit, i16 exactly, f16 as rounded from the oracle's f32) and the small batch,
  byte for byte, with the same chain results and the same exported stream states;
- every mapped window of the PCM arena, mirrors included, holds the sentinel outside the chains' write set, and the
  input arenas hold theirs outside what the test wrote;
- the batch ran on the path it was shaped for (expect_kernels)."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
import sparse_arena as sa
from helpers import (ALL_KERNELS, F32_GUARD, FRONT, GENERIC, I16_GUARD, RefStream, bits_equal, environ, expect_kernels, fill_guard,
                     launches_are_attributed, make_setup)
from lewton_b200 import _cabi as cabi
from test_async_batches import AsyncCall, Twin, check_arena, mappings, seq
from test_f16_output_gpu import F16_GUARD, same_f16
from test_f16_output_gpu import report as f16_report
from test_queued_batches import FLOOR, MIXED_EXTRA
from test_vq_shapes_gpu import Batch, Streams

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED
SPECTRUM, RESIDUE, HOST, DEVICE = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, cabi.MEM_DEVICE
MARGIN = 1 << 18              # elements mapped on each side of a span the batch touches

# setup kind: (channels, bs0, bs1, modes)
KINDS = {"mixed": (2, 8, 11, [(0, 0), (1, 0)]), "mid": (2, 10, 10, [(1, 0)]), "mid512": (2, 9, 9, [(1, 0)]),
         "short": (2, 8, 8, [(1, 0)]), "odd": (2, 6, 13, [(0, 0), (1, 0)]), "wide": (10, 8, 11, [(0, 0), (1, 0)])}
MIXED = {"k_long_s", "k_short_g"}
# path: (setup kind, sequence kind, packets per chain, entry, format, kernels that must run, kernels that may also run, env)
PATHS = {
    "long": ("mixed", "long", 8, SPECTRUM, F32P, {"k_long"}, set(), None),
    "long_residue": ("mixed", "long", 8, RESIDUE, I16P, FRONT | {"k_long"}, set(), None),
    "mid1024": ("mid", "uniform", 8, SPECTRUM, I16P, {"k_mid"}, set(), None),
    "mid512_residue": ("mid512", "uniform", 8, RESIDUE, F32P, FRONT | {"k_mid"}, set(), None),
    "short": ("short", "uniform", 16, SPECTRUM, F32P, {"k_short"}, set(), None),
    "segmented": ("mixed", "mixed", 16, SPECTRUM, F32P, MIXED, MIXED_EXTRA, None),
    "segmented_residue": ("mixed", "mixed", 16, RESIDUE, I16P, FRONT | {"k_long_s"}, MIXED | MIXED_EXTRA, None),
    "rounds": ("mixed", "mixed", 16, SPECTRUM, F32P, {"k_long", "k_short"}, {"k_chain", "k_row_copy"}, {"LWB_MIXED_ROUNDS": "1"}),
    "chain": ("odd", "mixed", 12, SPECTRUM, F32I, {"k_chain"}, set(), None),
    "chain_residue": ("mixed", "mixed", 12, RESIDUE, I16I, {"k_chain"}, set(), None),
    "generic": ("wide", "mixed", 6, SPECTRUM, F32P, GENERIC - {"k_prologue"}, set(), None),
    "generic_stereo": ("mixed", "mixed", 6, RESIDUE, F32P, GENERIC - {"k_prologue"} | FRONT, set(), {"LWB_FORCE_GENERIC": "1"}),
    "generic_residue": ("wide", "mixed", 6, RESIDUE, F32P, GENERIC, set(), None),     # > 8 channels: k_prologue
}
T32 = 1 << 32
# offset classes: A f32 bytes past 4 GiB, B negative as int32, C wraps as uint32, D a chain's range crosses 2^32
CLASS = {"0": 0, "A": (1 << 30) + 4, "B": (1 << 31) + 4, "C": T32 + 4, "D": T32 - 4096}
ROW_F = (1 << 30) + 4         # F: stereo packet rows whose row * C passes 2^31, and whose floor1_y words (row * C * LWB_MAX_POSTS) pass 2^32
ROW_W = (1 << 28) + 4         # F for 10 channels: row * C passes 2^31
STRIDE_E = T32 + 4            # E: planes 2^32 + 4 elements apart

# (path, coefficient class, PCM class, extra): extra may set "stride" (E), "rows" (F, with "floors" HOST / DEVICE)
CASES = [
    ("long", "C", "0", {}), ("long", "0", "C", {}), ("long", "B", "D", {}), ("long", "0", "0", {"stride": STRIDE_E}),
    ("long_residue", "A", "B", {"rows": ROW_F, "floors": HOST}), ("long_residue", "D", "C", {"rows": ROW_F, "floors": DEVICE}),
    ("mid1024", "C", "A", {}), ("mid1024", "0", "C", {"stride": STRIDE_E}),
    ("mid512_residue", "B", "C", {}), ("mid512_residue", "C", "D", {"rows": ROW_F, "floors": DEVICE}),
    ("short", "D", "B", {}), ("short", "A", "C", {}),
    ("segmented", "C", "C", {}), ("segmented", "A", "D", {"stride": STRIDE_E}),
    ("segmented_residue", "C", "B", {"rows": ROW_F, "floors": HOST}),
    ("rounds", "B", "C", {}),
    ("chain", "C", "C", {}), ("chain", "A", "D", {}),
    ("chain_residue", "D", "B", {"rows": ROW_F, "floors": DEVICE}),
    ("generic", "C", "C", {}), ("generic", "0", "B", {"stride": STRIDE_E}),
    ("generic_stereo", "B", "C", {"rows": ROW_F, "floors": HOST}),
    ("generic_residue", "C", "A", {"rows": ROW_W, "floors": DEVICE}), ("generic_residue", "A", "C", {"rows": ROW_W, "floors": HOST}),
]


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sus(ctx):
    return {k: make_setup(ctx, Cn, b0, b1, modes=m, mappings=mappings(Cn), floors=[FLOOR]) for k, (Cn, b0, b1, m) in KINDS.items()}


class KTwin(Twin):
    """A device stream and its oracle twin for a setup kind of KINDS."""

    def __init__(self, oracle, su, kind):
        Cn, self.bs0, self.bs1, self.modes = KINDS[kind]
        self.su, self.C = su, Cn
        self.pwr = L.PreviousWindowRight(su)
        self.ref = RefStream(oracle, Cn, self.bs0, self.bs1, self.modes, mappings(Cn), [FLOOR])


def planar(fmt):
    return fmt in (F32P, I16P, cabi.OUT_F16_PLANAR)


def spans(chains, channels, ns, fmt):
    """Per chain, the element spans it writes (include/lewton_b200.h, lwb_chain)."""
    out = []
    for c, Cn, n in zip(chains, channels, ns):
        out.append([(c.out_offset + k * c.out_stride, n) for k in range(Cn)] if planar(fmt) else [(c.out_offset, n * Cn)])
    return out


def build(ctx, oracle, sus, path, S, seed, memory, pinned=True):
    kind, seq_kind, P, entry, fmt, ran, extra, env = PATHS[path]
    rng = np.random.default_rng(seed)
    tws = [KTwin(oracle, sus[kind], kind) for _ in range(S)]
    call = AsyncCall(ctx, rng, [(tw, seq(rng, seq_kind, P)) for tw in tws], entry, fmt, memory,
                     (ran, ALL_KERNELS - ran - extra), pinned=pinned)
    return tws, call


class Large:
    """The batch of `call` moved: coefficients (and dense floors) by cshift elements, PCM by oshift, packet rows by rshift,
    planes `stride` apart; in sparse arenas of `memory`, floor arrays in sparse arenas of `floors`."""

    def __init__(self, ctx, call, cshift, oshift, rshift=0, stride=None, memory=DEVICE, floors=HOST):
        self.ctx, self.call, self.memory = ctx, call, memory
        fmt, residue = call.fmt, call.entry == RESIDUE
        self.channels = [tw.C for tw, _ in call.items]
        self.chains = []
        for c in call.chains:
            b = L.ChainSpec(c.pwr, c.modes, c.prev, c.next, coeff_offset=c.coeff_offset + cshift,
                            packet_index=c.packet_index + rshift, out_offset=c.out_offset + oshift,
                            out_stride=(stride or c.out_stride) if planar(fmt) else 0)
            self.chains.append(b)
        Arena = sa.DeviceArena if memory == DEVICE else sa.HostArena
        dt = call.pcm.dtype
        self.use(call)
        hi = max(lo + n for lo, n in self.write)
        self.pcm = Arena(dt, F32_GUARD if dt == np.float32 else I16_GUARD, hi + MARGIN)
        for lo, n in self.write:
            self.pcm.cover(max(0, lo - MARGIN), lo + n + MARGIN - max(0, lo - MARGIN))
        self.inputs = []                # (arena, element offset, array written there)
        self.coeffs = self.input(Arena, call.coeffs, cshift)
        self.dense = self.input(Arena, call.dense, cshift) if residue else None
        self.kinds = self.ys = None
        self.floor_memory = floors
        if residue:
            FA = sa.DeviceArena if floors == DEVICE else sa.HostArena
            Cn = self.channels[0]
            self.kinds = self.input(FA, call.kinds.ravel(), rshift * Cn, guard=0xFF)
            self.ys = self.input(FA, call.ys.ravel(), rshift * Cn * cabi.MAX_POSTS, guard=0xA5A5A5A5)
        for a in [self.pcm] + [x[0] for x in self.inputs]:
            a.commit(ctx)
        for a, off, arr in self.inputs:
            a.write(off, arr)

    def use(self, call):
        """Takes the outputs of `call` (same layout) as what the next run must write."""
        self.call = call
        self.ns = [w.shape[1] for w in call.wants]
        self.write = [s for sp in spans(self.chains, self.channels, self.ns, call.fmt) for s in sp]

    def input(self, Arena, arr, off, guard=F32_GUARD):
        a = Arena(arr.dtype, guard, off + arr.size + MARGIN)
        a.cover(max(0, off - MARGIN), off + arr.size + MARGIN - max(0, off - MARGIN))
        self.inputs.append((a, off, arr))
        return a

    def addr(self, a):
        if a is None:
            return None
        return a.ptr if isinstance(a, sa.DeviceArena) else a.arr

    def io_args(self):
        call = self.call
        kw = {}
        if call.entry == RESIDUE:
            kw = dict(floor_kind=self.addr(self.kinds), floor1_y=self.addr(self.ys), dense_floor=self.addr(self.dense),
                      floor_memory=self.floor_memory)
        return (self.chains, call.entry, self.memory, self.addr(self.coeffs), self.addr(self.pcm), call.fmt), kw

    def page_lock(self):
        """A host-memory submit's extent, page-locked (check_page_locked looks at the extent only)."""
        lo = min(c.coeff_offset for c in self.chains)
        self.coeffs.page_lock(lo, self.call.coeffs.size)
        if self.dense is not None:
            self.dense.page_lock(lo, self.call.dense.size)
        o_lo = min(lo for lo, _ in self.write)
        self.pcm.page_lock(o_lo, max(lo + n for lo, n in self.write) - o_lo)
        if self.kinds is not None and self.floor_memory == HOST:
            self.kinds.page_lock(self.inputs[-2][1], self.call.kinds.size)
            self.ys.page_lock(self.inputs[-1][1], self.call.ys.size)

    def compact(self):
        """The moved batch's PCM laid out as the small batch's arena: its write set copied to the small offsets."""
        call = self.call
        out = fill_guard(np.empty(call.total, call.pcm.dtype))
        small = spans(call.chains, self.channels, self.ns, call.fmt)
        big = spans(self.chains, self.channels, self.ns, call.fmt)
        for sp_s, sp_b in zip(small, big):
            for (ls, n), (lb, _) in zip(sp_s, sp_b):
                if n:
                    out[ls:ls + n] = self.pcm.read(lb, n)
        return out

    def check(self, oracle, small_pcm, what):
        self.ctx.synchronize()
        # the windows first: a truncated address shows up here as what it is, before the PCM it failed to write
        self.pcm.check_guard(self.write, (what, "pcm"))
        for a, off, arr in self.inputs:
            a.check_guard([(off, arr.size)], (what, "input"))
        got = self.compact()
        u = np.uint32 if got.dtype == np.float32 else np.uint16
        for a, b in zip(self.call.chains, self.chains):         # (check_arena takes the write set from the results)
            a.n_samples, a.packets_done, a.status = b.n_samples, b.packets_done, b.status
        check_arena(oracle, got, self.call.chains, self.call.wants, self.channels, self.call.fmt, what)
        if small_pcm is not None:
            assert np.array_equal(got.view(u), small_pcm.view(u)), (what, "PCM differs from the batch at small offsets")

    def physical_bytes(self):
        return sum(a.physical_bytes() for a in [self.pcm] + [x[0] for x in self.inputs])

    def close(self):
        self.ctx.synchronize()
        for a in [self.pcm] + [x[0] for x in self.inputs]:
            a.close()


def small_run(ctx, oracle, sus, path, seed, memory, how):
    """The batch at small offsets in ordinary arenas: its twins, call, PCM and final states."""
    tws, call = build(ctx, oracle, sus, path, 4, seed, memory)
    with environ(PATHS[path][7]):
        if how == "submit":
            call.submit(ctx)
            call.ticket.wait()
        else:
            call.decode(ctx)
    ctx.synchronize()                   # (a device-memory batch returns once queued)
    call.check(oracle, (path, "small"))
    pcm = call.dev["pcm"].cpu().numpy() if memory == DEVICE else call.pcm.copy()
    return tws, call, pcm


def compare(call_small, tws_small, large, tws, what):
    for a, b in zip(call_small.chains, large.chains):
        assert (a.status, a.packets_done, a.n_samples) == (b.status, b.packets_done, b.n_samples), what
    for ts, tb in zip(tws_small, tws):
        tb.check_state(what)
        a, b = ts.pwr.data(), tb.pwr.data()
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, "state differs from the small batch")


def run_large(ctx, large, call, how="decode", env=None):
    args, kw = large.io_args()
    ran, not_ran = call.expect
    with environ(env):
        with expect_kernels(ctx, ran=ran, not_ran=not_ran):
            if how == "submit":
                t = ctx.submit_chains(*args, **kw)
            else:
                L.decode_chains(ctx, *args, **kw)
    if how == "submit":
        t.wait()


@pytest.mark.parametrize("path,cc,oc,extra", CASES, ids=[f"{p}-c{c}-o{o}" + ("-E" if "stride" in x else "") +
                                                         ("-F" + ("dev" if x.get("floors") == DEVICE else "host") if "rows" in x else "")
                                                         for p, c, o, x in CASES])
def test_device_batch_at_large_offsets(ctx, oracle, sus, path, cc, oc, extra):
    seed = 7 + list(PATHS).index(path)
    tws_s, call_s, pcm_s = small_run(ctx, oracle, sus, path, seed, DEVICE, "decode")
    tws, call = build(ctx, oracle, sus, path, 4, seed, HOST, pinned=False)
    large = Large(ctx, call, CLASS[cc], CLASS[oc], extra.get("rows", 0), extra.get("stride"), DEVICE, extra.get("floors", HOST))
    try:
        assert large.physical_bytes() < (256 << 20)
        what = (path, cc, oc, extra)
        run_large(ctx, large, call, env=PATHS[path][7])
        large.check(oracle, pcm_s, what)
        compare(call_s, tws_s, large, tws, what)
    finally:
        large.close()


def test_misaligned_offset_falls_back_to_the_chain_kernel(ctx, oracle, sus):
    """A k_long batch whose PCM offset is 2 mod 4 at class C: the fused kernels' alignment is lost, k_chain takes it."""
    tws_s, call_s, pcm_s = small_run(ctx, oracle, sus, "long", 41, DEVICE, "decode")
    tws, call = build(ctx, oracle, sus, "long", 4, 41, HOST, pinned=False)
    call.expect = ({"k_chain"}, ALL_KERNELS - {"k_chain"})
    large = Large(ctx, call, CLASS["C"], T32 + 6)
    try:
        run_large(ctx, large, call)
        large.check(oracle, None, "misaligned")
        compare(call_s, tws_s, large, tws, "misaligned")
    finally:
        large.close()


@pytest.mark.parametrize("how", ["decode", "submit", "chunks"])
def test_host_batch_at_large_offsets(ctx, oracle, sus, how):
    """Host-memory batches at class C, in pageable sparse host arenas: lwb_decode_chains, lwb_submit_chains (the extent
    page-locked) and three chunks (LWB_E2E_CHUNKS=3), on the residue entry with host floors at packet row 2^30 + 4."""
    path = "segmented_residue" if how == "chunks" else "long_residue"
    seed = 50 + ["decode", "submit", "chunks"].index(how)
    env = {"LWB_E2E_CHUNKS": "3"} if how == "chunks" else None
    with environ(env):
        tws_s, call_s, pcm_s = small_run(ctx, oracle, sus, path, seed, HOST, "submit" if how == "submit" else "decode")
    tws, call = build(ctx, oracle, sus, path, 4, seed, HOST, pinned=False)
    large = Large(ctx, call, CLASS["C"], CLASS["C"], ROW_F, None, HOST, HOST)
    try:
        if how == "submit":
            large.page_lock()
        run_large(ctx, large, call, "submit" if how == "submit" else "decode", env)
        large.check(oracle, pcm_s, ("host", how))
        compare(call_s, tws_s, large, tws, ("host", how))
    finally:
        large.close()


def prepared_runs(ctx, oracle, sus, moved):
    """An lwb_plan of a k_long batch, run twice on the next packets of its streams (planned, then planned again: the
    streams changed shape), at small offsets in ordinary device arenas or (moved) at class C in sparse ones.  Per run the
    PCM in the small layout and the chain results, checked against the oracle; then the final states."""
    kind, seq_kind, P, entry, fmt, ran, _, _ = PATHS["long"]
    rng = np.random.default_rng(61)
    tws = [KTwin(oracle, sus[kind], kind) for _ in range(4)]
    items = [(tw, seq(rng, seq_kind, P)) for tw in tws]
    calls = [AsyncCall(ctx, rng, items, entry, fmt, HOST if moved else DEVICE, (ran, ALL_KERNELS - ran), pinned=False) for _ in range(2)]
    out = []
    large = Large(ctx, calls[0], CLASS["C"], CLASS["C"]) if moved else None
    try:
        if moved:
            args, kw = large.io_args()
        else:
            args, kw = (calls[0].chains, entry, DEVICE, *calls[0].arenas(), fmt), {}
        batch = L.Batch(ctx, *args, **kw)
        for k, call in enumerate(calls):
            ctx.synchronize()
            if k and moved:
                large.coeffs.write(large.chains[0].coeff_offset, call.coeffs)
                for a, b in large.pcm.windows:          # the sentinel again
                    ctx.h2d(large.pcm.res + a, large.pcm._guard_words(b - a))
                large.use(call)
            elif k:
                calls[0].dev["coeffs"].copy_(call.dev["coeffs"])
                calls[0].dev["pcm"].copy_(call.dev["pcm"])      # (the sentinel)
                torch.cuda.synchronize()
            with expect_kernels(ctx, ran={"k_long": 1}, not_ran=ALL_KERNELS - {"k_long"}):
                batch.run()
            batch.collect()
            ctx.synchronize()
            if moved:
                large.check(oracle, None, ("prepared", k))
                pcm = large.compact()
            else:
                pcm = calls[0].dev["pcm"].cpu().numpy()
                for a, b in zip(call.chains, calls[0].chains):
                    a.n_samples, a.packets_done, a.status = b.n_samples, b.packets_done, b.status
                check_arena(oracle, pcm, call.chains, call.wants, [tw.C for tw in tws], fmt, ("prepared small", k))
            out.append((pcm, [(c.n_samples, c.packets_done, c.status) for c in batch.chains]))
        batch.close()
    finally:
        if large:
            large.close()
    for tw in tws:                                      # (the twins ran both calls' packets when they were built)
        tw.check_state(("prepared", moved))
    return out, [tw.pwr.data() for tw in tws]


def test_prepared_batch_at_large_offsets(ctx, oracle, sus):
    """The plan at class C against the oracle, its sentinels and, run by run, the same plan at small offsets: the same PCM
    bytes and chain results, and the same final states."""
    small, s_states = prepared_runs(ctx, oracle, sus, False)
    big, b_states = prepared_runs(ctx, oracle, sus, True)
    for k, ((ps, rs), (pb, rb)) in enumerate(zip(small, big)):
        assert rs == rb, ("prepared", k, "chain results")
        assert ps.view(np.uint32).tobytes() == pb.view(np.uint32).tobytes(), ("prepared", k, "PCM differs from the small plan")
    for a, b in zip(s_states, b_states):
        assert bits_equal(a, b), "prepared: state differs from the small plan"


# ---------------------------------------------------------------------------------------------------------------------
# packer bitstreams: VQ runs and entries past 2^32 (class G), floor-0 records at packet rows past 2^30 (class F), f16
# ---------------------------------------------------------------------------------------------------------------------
VQ, F16P, F16I = cabi.ENTRY_VQ, cabi.OUT_F16_PLANAR, cabi.OUT_F16_INTERLEAVED
DTYPES = {F32P: np.float32, F32I: np.float32, I16P: np.int16, I16I: np.int16, F16P: np.float16, F16I: np.float16}
GUARD = {np.dtype(np.float32): F32_GUARD, np.dtype(np.int16): I16_GUARD, np.dtype(np.float16): F16_GUARD}
G = T32 + 4                   # G: VQ run and entry offsets past 2^32
# name: (channels, bs0, bs1, residue type, entry, format, memory, floor / VQ memory, shifts {c, o, r, v, e})
PACKER = {
    "vq_mid": (2, 10, 10, 1, VQ, F32P, DEVICE, DEVICE, dict(o=CLASS["C"], r=ROW_F, v=G, e=G)),
    "vq_chain": (2, 8, 11, 2, VQ, I16I, DEVICE, HOST, dict(o=CLASS["D"], r=ROW_F, v=G, e=CLASS["B"])),
    "vq_host": (2, 10, 10, 0, VQ, F16I, HOST, HOST, dict(o=CLASS["C"], r=ROW_F, v=CLASS["B"], e=G)),
    "residue_f16": (2, 10, 10, 0, RESIDUE, F16P, DEVICE, HOST, dict(c=CLASS["C"], o=CLASS["B"], r=ROW_F)),
}


def packer_kernels(entry, fmt, floor_mem, has_records):
    """(ran, not_ran): interleaved output on k_chain, planar 1024-point blocks through the front stages and k_mid; the
    floor-0 curves whenever the batch may carry records (device floor arrays cannot be looked at)."""
    f0 = {"k_floor0_curves": 1 if floor_mem == DEVICE or has_records else 0}
    if not planar(fmt):
        return {"k_chain": 1, **f0}, ALL_KERNELS - {"k_chain", "k_floor0_curves"}
    return {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_mid": 1, **f0}, ALL_KERNELS - FRONT - {"k_mid", "k_floor0_curves"}


class PackerRun:
    """One lwb_decode_chains of packer batch b (test_vq_shapes_gpu.Batch) with every offset moved by `sh` (c: coefficient
    elements, o: PCM elements, r: packet rows, v: VQ runs, e: VQ entries) in sparse arenas, or, sh None, in ordinary ones."""

    def __init__(self, ctx, b, entry, fmt, memory, floor_mem, sh):
        self.ctx, self.b, self.fmt, self.sparse = ctx, b, fmt, sh is not None
        sh = sh or {}
        c_sh, self.o_sh, r_sh, v_sh, e_sh = (sh.get(k, 0) for k in "corve")
        Cn, dt = b.st.C, np.dtype(DTYPES[fmt])
        self.ns = [w.shape[1] for w in b.wants]
        self.layout = [(m, p, n, c0 + c_sh, r + r_sh, o + self.o_sh, sd) for m, p, n, c0, r, o, sd in b.layout]
        runs, roffs, ents, eoffs = b.vq
        arrays = {"kinds": (b.kinds.ravel(), r_sh * Cn, 0xFF), "ys": (b.ys.ravel(), r_sh * Cn * cabi.MAX_POSTS, 0xA5A5A5A5)}
        if entry == VQ:
            arrays.update(roffs=(roffs + np.uint64(v_sh), r_sh, 0xA5A5A5A5A5A5A5A5), eoffs=(eoffs + np.uint64(e_sh), r_sh, 0xA5A5A5A5A5A5A5A5),
                          runs=(runs.view(np.uint64), v_sh, 0xA5A5A5A5A5A5A5A5), ents=(ents, e_sh, 0xA5A5))
        big = {"coeffs": (b.coeffs, c_sh, F32_GUARD)} if entry == RESIDUE else {}
        if b.dense is not None:
            big["dense"] = (b.dense, c_sh, F32_GUARD)
        self.write = [(o + k * sd, n) if planar(fmt) else (o, n * Cn) for (_, _, _, _, _, o, sd), n in zip(self.layout, self.ns)
                      for k in range(Cn if planar(fmt) else 1)]
        self.inputs, self.frees, self.ptr = [], [], {}
        for names, mem in ((arrays, floor_mem), (big, memory)):
            for name, (arr, off, guard) in names.items():
                self.ptr[name] = self.place(mem, arr, off, guard)
        hi = max(lo + n for lo, n in self.write)
        if self.sparse:
            self.pcm = (sa.DeviceArena if memory == DEVICE else sa.HostArena)(dt, GUARD[dt], hi + MARGIN)
            for lo, n in self.write:
                self.pcm.cover(max(0, lo - MARGIN), lo + n + MARGIN - max(0, lo - MARGIN))
            self.pcm.commit(ctx)
            self.ptr["pcm"] = self.pcm.ptr if memory == DEVICE else self.pcm.arr
        else:
            self.host_pcm = np.empty(b.n_out, dt)
            self.host_pcm.view(sa._UINT[dt.itemsize])[...] = GUARD[dt]
            self.ptr["pcm"] = self.dev(self.host_pcm) if memory == DEVICE else self.host_pcm
        for a, off, arr in self.inputs:
            a.write(off, arr)
        self.entry, self.memory, self.floor_mem = entry, memory, floor_mem

    def dev(self, a):
        p = self.ctx.device_alloc(max(a.nbytes, 16))
        self.ctx.h2d(p, a)
        self.frees.append(p)
        return p

    def place(self, mem, arr, off, guard):
        arr = np.ascontiguousarray(arr)
        if not self.sparse:
            return self.dev(arr) if mem == DEVICE else arr
        a = (sa.DeviceArena if mem == DEVICE else sa.HostArena)(arr.dtype, guard, off + arr.size + MARGIN)
        a.cover(max(0, off - MARGIN), off + arr.size + MARGIN - max(0, off - MARGIN))
        a.commit(self.ctx)
        self.inputs.append((a, off, arr))
        return a.ptr if mem == DEVICE else a.arr

    def run(self, pwrs, expect):
        p = self.ptr
        self.chains = [L.ChainSpec(pwrs[s], m, pv, n, coeff_offset=c0, packet_index=r, out_offset=o, out_stride=sd)
                       for s, (m, pv, n, c0, r, o, sd) in enumerate(self.layout)]
        kw = dict(floor_kind=p["kinds"], floor1_y=p["ys"], dense_floor=p.get("dense"), floor_memory=self.floor_mem)
        if self.entry == VQ:
            kw["vq"] = (p["runs"], p["roffs"], p["ents"], p["eoffs"])
        with expect_kernels(self.ctx, *expect):
            L.decode_chains(self.ctx, self.chains, self.entry, self.memory, p.get("coeffs"), p["pcm"], self.fmt, **kw)
        self.ctx.synchronize()

    def pcm_small_layout(self):
        """The PCM laid out as the batch at small offsets (its write set; the sentinel elsewhere)."""
        if not self.sparse:
            if self.memory == DEVICE:
                self.ctx.d2h(self.host_pcm, self.ptr["pcm"])
            return self.host_pcm.copy()
        dt = self.pcm.dtype
        out = np.empty(self.b.n_out, dt)
        out.view(sa._UINT[dt.itemsize])[...] = GUARD[dt]
        for lo, n in self.write:
            out[lo - self.o_sh:lo - self.o_sh + n] = self.pcm.read(lo, n)
        return out

    def check(self, oracle, what):
        """Sentinels (every window, mirrors included), then every chain against the oracle; returns the PCM."""
        if self.sparse:
            self.pcm.check_guard(self.write, (what, "pcm"))
            for a, off, arr in self.inputs:
                a.check_guard([(off, arr.size)], (what, "input"))
        pcm = self.pcm_small_layout()
        Cn = self.b.st.C
        mask = np.zeros(pcm.size, bool)
        for s, (w, c) in enumerate(zip(self.b.wants, self.chains)):
            n = w.shape[1]
            assert (c.status, c.packets_done, c.n_samples) == (0, len(c.modes), n), (what, s, c.status, c.n_samples, n)
            _, _, _, _, _, o, sd = self.b.layout[s]
            got = pcm[o:o + Cn * sd].reshape(Cn, sd)[:, :n] if planar(self.fmt) else pcm[o:o + n * Cn].reshape(n, Cn).T
            if planar(self.fmt):
                for k in range(Cn):
                    mask[o + k * sd:o + k * sd + n] = True
            else:
                mask[o:o + n * Cn] = True
            if pcm.dtype == np.float32:
                assert bits_equal(got, w), (what, s)
            elif pcm.dtype == np.int16:
                assert np.array_equal(got, oracle.quantise_i16(w)), (what, s)
            else:
                assert same_f16(got, w), (what, s, f16_report(got, w))
        u = sa._UINT[pcm.dtype.itemsize]
        assert not np.any(~mask & (pcm.view(u) != GUARD[pcm.dtype])), (what, "written outside the write set")
        return pcm

    def close(self):
        self.ctx.synchronize()
        for p in self.frees:
            self.ctx.device_free(p)
        for a in [x[0] for x in self.inputs] + ([self.pcm] if self.sparse else []):
            a.close()


@pytest.mark.parametrize("name", list(PACKER))
def test_packer_batch_at_large_offsets(ctx, oracle, name):
    """Packer streams with floor-0 records (k_floor0_curves reads their floor1_y rows at packet row 2^30 + 4), on the VQ
    entry with run and entry offsets moved past 2^31 or 2^32 and on the residue entry; f32, i16 and f16 output.  The moved
    batch against the oracle and byte for byte against the same batch at small offsets, with the same chain results and
    stream states."""
    Cn, bs0, bs1, rtype, entry, fmt, memory, floor_mem, sh = PACKER[name]
    S, P = 3, 6
    st = Streams(4200 + list(PACKER).index(name), Cn, bs0, bs1, rtype, True, S, P, p_short=0.1)
    su = st.hdr.make_setup(ctx, floor0=True)
    b = Batch(st, 0, P, F32P if planar(fmt) else F32I, st.twins(oracle))   # (the layout, in elements, of either format)
    assert b.has_records, "no floor-0 record in the batch"
    expect = packer_kernels(entry, fmt, floor_mem, b.has_records)
    outs, states, results = [], [], []
    for moved in (None, sh):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        r = PackerRun(ctx, b, entry, fmt, memory, floor_mem, moved)
        try:
            r.run(pwrs, expect)
            outs.append(r.check(oracle, (name, "moved" if moved else "small")))
            results.append([(c.status, c.packets_done, c.n_samples) for c in r.chains])
            states.append([p.data() for p in pwrs])
        finally:
            r.close()
            for p in pwrs:
                p.close()
    assert outs[0].tobytes() == outs[1].tobytes(), (name, "PCM differs from the batch at small offsets")
    assert results[0] == results[1], name
    for a, bb in zip(*states):
        assert (a is None) == (bb is None) and (a is None or bits_equal(a, bb)), (name, "state differs from the small batch")
