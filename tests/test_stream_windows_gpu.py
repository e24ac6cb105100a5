"""Output windows (lwb_stream_set_window) on the GPU.  A windowed stream writes exactly the samples of its window: each
chain's n_samples is what it wrote, its written samples equal the oracle's full decode sliced to the window (f32 bit for
bit; i16 and f16 exactly as the unwindowed decode gives them), every element outside the written set keeps its
sentinel, and the stream states are those of the unwindowed decode.  Windows span batches (skips inside the first
packet, over whole chains and batches; limits ending mid-packet or used up before a chain starts) on every batch path,
entry, format and memory space, through lwb_decode_chains, two-deep lwb_submit_chains and prepared batches.  A batch
with clipped chains launches exactly the kernels of the same batch without windows, plus one k_row_copy."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import RefStream, bits_equal, environ, expect_kernels, launches_are_attributed, make_setup, mismatch_report, random_floor1_y

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
F32P, I16P, F32I, I16I, F16P, F16I = (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED,
                                      cabi.OUT_F16_PLANAR, cabi.OUT_F16_INTERLEAVED)
DTYPE = {F32P: np.float32, F32I: np.float32, I16P: np.int16, I16I: np.int16, F16P: np.float16, F16I: np.float16}
PLANAR = (F32P, I16P, F16P)
GUARD = {4: 0x7fa5a5a5, 2: 0x5a5a}
SPECTRUM, RESIDUE = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE

# path: (channels, blocksize_0, blocksize_1, share of short blocks, environment, the kernel that must run)
PATHS = {
    "k_long": (2, 8, 11, 0.0, None, "k_long"),
    "k_mid_1024": (2, 8, 10, 0.0, None, "k_mid"),
    "k_mid_512": (2, 8, 9, 0.0, None, "k_mid"),
    "one_pass": (2, 8, 11, 0.3, None, "k_long_s"),
    "rounds": (2, 8, 11, 0.3, {"LWB_MIXED_ROUNDS": "1"}, "k_short"),
    "k_chain": (2, 8, 11, 0.3, {"LWB_FORCE_GENERIC": "chain"}, "k_chain"),
    "four_kernel": (2, 8, 11, 0.3, {"LWB_FORCE_GENERIC": "1"}, "k_imdct"),
}


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def flags(bf):
    n = len(bf)
    prev, nxt = np.ones(n, np.uint8), np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


class Stream:
    """A windowed stream, its unwindowed twin (same setup, same packets) and, optionally, its oracle twin."""

    def __init__(self, su, oracle, C, bs0, bs1, bf, window):
        self.su, self.C, self.bs0, self.bs1 = su, C, bs0, bs1
        self.win, self.full = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
        self.ref = RefStream(oracle, C, bs0, bs1, [(0, 0), (1, 0)], [{"coupling": [(0, 1)] if C == 2 else [], "floor_of_channel": [0] * C}],
                             [FLOOR]) if oracle is not None else None
        self.bf = bf
        self.prev, self.nxt = flags(bf)
        self.at = 0                    # packets taken
        self.pos = 0                   # samples produced so far
        self.window = window           # (skip, limit or None), or None: no window
        if window:
            self.win.set_window(*window)
        self.oracle_pcm = []

    def expect(self, n):
        """The [a, b) of the next n produced samples that the window writes."""
        if not self.window:
            return 0, n
        skip, limit = self.window
        end = np.inf if limit is None else skip + limit
        a = int(min(max(skip - self.pos, 0), n))
        b = int(max(a, min(end - self.pos, n)))
        return a, b


def make_packets(rng, st, k, entry):
    """Inputs of the next k packets of st: (modes, prev, next, coeffs [rows], kinds, ys, dense, produced samples)."""
    sl = slice(st.at, st.at + k)
    bf, prev, nxt = st.bf[sl], st.prev[sl], st.nxt[sl]
    st.at += k
    has = not st.full.is_empty()
    n = 0
    coeffs, kinds, ys, dense = [], [], [], []
    for i in range(len(bf)):
        if has:
            n += L.get_decoded_sample_count(st.su, int(bf[i]), int(prev[i]), int(nxt[i]))
        has = True
        n2 = (1 << (st.bs1 if bf[i] else st.bs0)) // 2
        if entry == RESIDUE:
            res = (rng.standard_normal((st.C, n2)) * rng.integers(0, 2, (st.C, n2))).astype(np.float32)
            fl = [None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.2 else random_floor1_y(rng, FLOOR[0], len(FLOOR[1]))
                  for r in rng.random(st.C)]
            kd, y, d = L.DecodedPacket(int(bf[i]), res, fl).pack()
            kinds.append(kd)
            ys.append(y)
            dense.append(np.zeros_like(res) if d is None else d)
            if st.ref:
                rc, o = st.ref.packet(int(bf[i]), int(prev[i]), int(nxt[i]), res, fl)
        else:
            res = (rng.standard_normal((st.C, n2)) * 0.1).astype(np.float32)
            if st.ref:
                rc, o = st.ref.spectrum(int(bf[i]), int(prev[i]), int(nxt[i]), res)
        if st.ref:
            assert rc == 0
            st.oracle_pcm.append(o)
        coeffs.append(res.ravel())
    return bf, prev, nxt, coeffs, kinds, ys, dense, n


class Arena:
    """A PCM arena in host or device memory, filled with the sentinel; `shift` bytes past a 16-byte boundary."""

    def __init__(self, ctx, n_elems, fmt, memory, shift=0, pinned=False):
        self.esz = np.dtype(DTYPE[fmt]).itemsize
        self.nbytes, self.shift, self.memory = n_elems * self.esz, shift, memory
        img = np.zeros(self.nbytes // self.esz, np.uint32 if self.esz == 4 else np.uint16)
        img[...] = GUARD[self.esz]
        self.image = img.view(np.uint8)
        if memory == cabi.MEM_DEVICE:
            self.t = torch.empty(self.nbytes + 32, dtype=torch.uint8, device="cuda")
            self.t[shift:shift + self.nbytes].copy_(torch.from_numpy(self.image.copy()))
            torch.cuda.synchronize()
            self.ptr = self.t.data_ptr() + shift
        else:
            self.h = ctx.host_alloc(self.nbytes + 32, np.uint8) if pinned else np.zeros(self.nbytes + 32, np.uint8)
            self.h[shift:shift + self.nbytes] = self.image
            self.ptr = self.h[shift:]

    def read(self):
        if self.memory == cabi.MEM_DEVICE:
            torch.cuda.synchronize()
            return self.t[self.shift:self.shift + self.nbytes].cpu().numpy()
        return np.array(self.h[self.shift:self.shift + self.nbytes])


def deinterleave(buf, fmt, K, n):
    """[K][n] of a chain's n samples at the start of buf."""
    return buf[:K * n].reshape(K, n) if fmt in PLANAR else buf[:n * K].reshape(n, K).T


class Batch:
    """One batch over streams: every stream's next k packets, laid out once for the windowed and once for the unwindowed
    twins.  The windowed chains' planes sit `odd` elements off a multiple of 4 (0: aligned), padded."""

    def __init__(self, rng, streams, k, entry, fmt, odd=0):
        self.entry, self.fmt = entry, fmt
        self.parts = [make_packets(rng, st, k, entry) for st in streams]
        self.streams = streams
        self.coeffs = np.concatenate([c for p in self.parts for c in p[3]]).astype(np.float32)
        if entry == RESIDUE:
            self.kinds = np.ascontiguousarray(np.concatenate([np.stack(p[4]) for p in self.parts]))
            self.ys = np.ascontiguousarray(np.concatenate([np.stack(p[5]) for p in self.parts]))
            self.dense = np.concatenate([d.ravel() for p in self.parts for d in p[6]]).astype(np.float32)
        self.K = [st.su.output_channels for st in streams]
        # layouts: the twin tight, the windowed one padded and shifted
        self.full_lay, self.win_lay = [], []
        fo = wo = 0
        for i, p in enumerate(self.parts):
            n, K = p[7], self.K[i]
            self.full_lay.append((fo, n))
            fo += K * n
            stride = n + 4 + (odd and int(rng.integers(0, 3)))
            off = wo + odd
            self.win_lay.append((off, stride))
            wo = off + (K * stride if fmt in PLANAR else K * n) + 4
        self.full_elems, self.win_elems = max(fo, 1), wo + 8

    def chains(self, which, lay):
        out, co, pi = [], 0, 0
        for i, (st, p) in enumerate(zip(self.streams, self.parts)):
            bf, prev, nxt = p[0], p[1], p[2]
            off, stride = lay[i]
            out.append(L.ChainSpec(getattr(st, which), bf, prev, nxt, coeff_offset=co, packet_index=pi, out_offset=off, out_stride=stride))
            co += sum(c.size for c in p[3])
            pi += len(bf)
        return out

    def io(self):
        if self.entry == RESIDUE:
            return dict(floor_kind=self.kinds, floor1_y=self.ys, dense_floor=self.dense)
        return {}


def decode(ctx, b, which, memory, arena, chains, coeffs=None):
    kw = b.io()
    co = b.coeffs if coeffs is None else coeffs
    if memory == cabi.MEM_DEVICE:
        dco = torch.from_numpy(co).cuda()
        dden = torch.from_numpy(kw["dense_floor"]).cuda() if "dense_floor" in kw else None
        if dden is not None:
            kw["dense_floor"] = dden.data_ptr()
        torch.cuda.synchronize()
        L.decode_chains(ctx, chains, b.entry, memory, dco.data_ptr(), arena.ptr, b.fmt, **kw)
        torch.cuda.synchronize()
        return
    L.decode_chains(ctx, chains, b.entry, memory, co, arena.ptr, b.fmt, **kw)


def check_batch(b, full_chains, win_chains, full_buf, win_buf):
    """The windowed arena holds exactly the window of the unwindowed decode, and the sentinel elsewhere; returns the
    written counts.  Advances the streams' produced-sample counters."""
    esz = np.dtype(DTYPE[b.fmt]).itemsize
    want = np.zeros_like(win_buf)
    want.view(np.uint32 if esz == 4 else np.uint16)[...] = GUARD[esz]
    fv = full_buf.view(DTYPE[b.fmt])
    wv = want.view(DTYPE[b.fmt])
    counts = []
    for i, st in enumerate(b.streams):
        n, K = b.parts[i][7], b.K[i]
        fc, wc = full_chains[i], win_chains[i]
        assert fc.n_samples == n
        a, e = st.expect(n)
        assert wc.n_samples == e - a, (i, st.window, st.pos, n, wc.n_samples, (a, e))
        assert wc.packets_done == fc.packets_done and wc.status == fc.status == 0
        fo, _ = b.full_lay[i]
        full = deinterleave(fv[fo:], b.fmt, K, n)
        off, stride = b.win_lay[i]
        sl = full[:, a:e]
        if b.fmt in PLANAR:
            for k in range(K):
                wv[off + k * stride: off + k * stride + (e - a)] = sl[k]
        else:
            wv[off: off + (e - a) * K] = sl.T.ravel()
        st.pos += n
        counts.append(e - a)
    got = win_buf.view(np.uint32 if esz == 4 else np.uint16)
    exp = want.view(np.uint32 if esz == 4 else np.uint16)
    bad = np.nonzero(got != exp)[0]
    assert not bad.size, f"{bad.size} elements differ; first at element {bad[:5]}: got {got[bad[:5]]} want {exp[bad[:5]]}"
    return counts


def check_oracle_and_states(streams, full_pcm_by_stream, fmt):
    for st in streams:
        assert bits_equal(st.win.data() if not st.win.is_empty() else np.zeros(0), st.full.data() if not st.full.is_empty() else np.zeros(0))
        assert st.win.is_empty() == st.full.is_empty() and len(st.win) == len(st.full)
    if fmt not in (F32P, F32I):
        return
    for st, got in zip(streams, full_pcm_by_stream):
        if st.ref is None:
            continue
        want = np.concatenate(st.oracle_pcm, axis=1) if st.oracle_pcm else np.zeros((st.C, 0), np.float32)
        assert bits_equal(got, want), mismatch_report(got, want)


WINDOWS = [(100, None), None, (0, 1500), (3000, 40), (1700, 2600), (5000, None), (0, 10), (700, 0)]


def make_streams(ctx, oracle, rng, path, n_streams, total_packets, windows=WINDOWS, mix=None):
    C, bs0, bs1, p_short, _, _ = PATHS[path]
    su = make_setup(ctx, C, bs0, bs1, mappings=[{"coupling": [(0, 1)] if C == 2 else [], "floor_of_channel": [0] * C}], floors=[FLOOR])
    if mix is not None:
        su.set_output_mix(mix)
    out = []
    for i in range(n_streams):
        bf = (rng.random(total_packets) >= p_short).astype(np.uint8)
        out.append(Stream(su, oracle if mix is None else None, C, bs0, bs1, bf, windows[i % len(windows)]))
    return out


def run(ctx, oracle, path, memory, entry, fmt, n_batches=3, k=4, n_streams=8, odd=0, seed=0, mix=None, prove_kernels=True, shift=0, kernel=None,
        chunks=1):
    """chunks: the chunks a host-memory batch runs in (LWB_E2E_CHUNKS); one k_row_copy per chunk that moves samples."""
    rng = np.random.default_rng(seed)
    streams = make_streams(ctx, oracle, rng, path, n_streams, n_batches * k, mix=mix)
    env = dict(PATHS[path][4] or {}, **({"LWB_E2E_CHUNKS": str(chunks)} if chunks > 1 else {}))
    full_pcm = [[] for _ in streams]
    for bi in range(n_batches):
        b = Batch(rng, streams, k, entry, fmt, odd)
        fa = Arena(ctx, b.full_elems, fmt, memory)
        wa = Arena(ctx, b.win_elems, fmt, memory, shift=shift)
        fch, wch = b.chains("full", b.full_lay), b.chains("win", b.win_lay)
        with environ(env):
            with expect_kernels(ctx) as kfull:
                decode(ctx, b, "full", memory, fa, fch)
            with expect_kernels(ctx) as kwin:
                decode(ctx, b, "win", memory, wa, wch)
        fbuf, wbuf = fa.read(), wa.read()
        clipped = [st.window is not None and st.expect(p[7]) != (0, p[7]) for st, p in zip(streams, b.parts)]
        moves = [c and st.expect(p[7])[1] > st.expect(p[7])[0] for c, st, p in zip(clipped, streams, b.parts)]
        n = len(moves)
        row_copies = sum(any(moves[n * q // chunks:n * (q + 1) // chunks]) for q in range(chunks))
        for i, p in enumerate(b.parts):
            full_pcm[i].append(deinterleave(fbuf.view(DTYPE[fmt])[b.full_lay[i][0]:], fmt, b.K[i], p[7]).astype(np.float32))
        check_batch(b, fch, wch, fbuf, wbuf)
        if prove_kernels:
            assert kfull[kernel or PATHS[path][5]] > 0, kfull
            want = dict(kfull)
            want["k_row_copy"] += row_copies
            assert kwin == want, (kfull, kwin)
    check_oracle_and_states(streams, [np.concatenate(p, axis=1) for p in full_pcm], fmt)
    for st in streams:
        if st.window:
            skip, limit = st.window
            left = st.win.window
            assert left[0] == max(skip - st.pos, 0)
            assert left[1] == (None if limit is None else max(0, min(limit, skip + limit - st.pos)))
    return streams


@pytest.mark.parametrize("entry", [SPECTRUM, RESIDUE], ids=["spectrum", "residue"])
@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("path", list(PATHS))
def test_windows_on_every_path(ctx, oracle, path, memory, entry):
    run(ctx, oracle, path, memory, entry, F32P)


@pytest.mark.parametrize("path", ["k_long", "one_pass"])
def test_windows_in_chunked_host_batches(ctx, oracle, path):
    """A host-memory batch in three chunks (LWB_E2E_CHUNKS=3): each chunk moves its clipped chains' samples behind its
    own kernels, one k_row_copy per chunk with samples to move, before its PCM goes home."""
    run(ctx, oracle, path, cabi.MEM_HOST, RESIDUE, F32P, seed=8, chunks=3, n_streams=9)


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("fmt", [F32P, I16P, F16P, F32I, I16I, F16I], ids=["f32p", "i16p", "f16p", "f32i", "i16i", "f16i"])
def test_windows_in_every_format(ctx, oracle, fmt, memory):
    run(ctx, oracle, "k_long" if fmt in PLANAR else "k_chain", memory, RESIDUE, fmt, seed=1)


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
def test_windows_with_an_output_mix(ctx, oracle, memory):
    mix = np.array([[0.5, 0.5], [0.0, 1.0], [1.0, 0.0]], np.float32)
    run(ctx, oracle, "k_long", memory, SPECTRUM, F32P, mix=mix, seed=2, kernel="k_chain")     # (a mix runs on k_chain)


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("fmt", [F32P, I16P, F16I], ids=["f32p", "i16p", "f16i"])
def test_unaligned_offsets(ctx, oracle, fmt, memory):
    """Windowed chains at element offsets off every multiple of 4, in an arena one or three elements past a 16-byte
    boundary: k_row_copy stores them between any two element-aligned addresses (the batch's path may differ from the
    aligned one's)."""
    esz = np.dtype(DTYPE[fmt]).itemsize
    run(ctx, oracle, "k_long", memory, SPECTRUM, fmt, odd=1, seed=3, prove_kernels=False, shift=esz if memory == cabi.MEM_DEVICE else 3 * esz)


def test_every_chain_clipped_keeps_the_fused_kernel(ctx, oracle):
    """Every chain clipped at both ends, at offsets that are not multiples of 4: their full outputs sit in aligned
    scratch, so the batch still runs on k_long, plus one k_row_copy."""
    rng = np.random.default_rng(4)
    streams = make_streams(ctx, oracle, rng, "k_long", 6, 4, windows=[(300, 2000), (1, 3000), (1023, 1)])
    b = Batch(rng, streams, 4, SPECTRUM, F32P, odd=1)
    fa, wa = Arena(ctx, b.full_elems, F32P, cabi.MEM_DEVICE), Arena(ctx, b.win_elems, F32P, cabi.MEM_DEVICE)
    fch, wch = b.chains("full", b.full_lay), b.chains("win", b.win_lay)
    with expect_kernels(ctx, ran={"k_long": 1}):
        decode(ctx, b, "full", cabi.MEM_DEVICE, fa, fch)
    with expect_kernels(ctx, ran={"k_long": 1, "k_row_copy": 1, "k_chain": 0}):
        decode(ctx, b, "win", cabi.MEM_DEVICE, wa, wch)
    check_batch(b, fch, wch, fa.read(), wa.read())


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
def test_two_deep_submits(ctx, oracle, memory):
    """Batches queued two deep before their tickets are waited on: the windows move at submit time."""
    rng = np.random.default_rng(5)
    streams = make_streams(ctx, oracle, rng, "one_pass", 8, 12)
    batches, pending = [], []
    for bi in range(3):
        b = Batch(rng, streams, 4, SPECTRUM, F32P)
        fa = Arena(ctx, b.full_elems, F32P, memory, pinned=True)
        wa = Arena(ctx, b.win_elems, F32P, memory, pinned=True)
        fch, wch = b.chains("full", b.full_lay), b.chains("win", b.win_lay)
        keep = []
        for which, ar, ch in (("full", fa, fch), ("win", wa, wch)):
            if memory == cabi.MEM_DEVICE:
                dco = torch.from_numpy(b.coeffs).cuda()
                keep.append(dco)
                torch.cuda.synchronize()
                t = ctx.submit_chains(ch, SPECTRUM, memory, dco.data_ptr(), ar.ptr, F32P)
            else:
                co = ctx.host_alloc(b.coeffs.size, np.float32)
                co[...] = b.coeffs
                keep.append(co)
                t = ctx.submit_chains(ch, SPECTRUM, memory, co, ar.ptr, F32P)
            pending.append(t)
        batches.append((b, fa, wa, fch, wch, keep))
        if bi >= 1:                          # two batches in flight
            b0, fa0, wa0, fch0, wch0, _ = batches[bi - 1]
            for t in pending[:2]:
                t.wait()
            pending = pending[2:]
            check_batch(b0, fch0, wch0, fa0.read(), wa0.read())
    for t in pending:
        t.wait()
    b, fa, wa, fch, wch, _ = batches[-1]
    check_batch(b, fch, wch, fa.read(), wa.read())
    check_oracle_and_states(streams, [], F32P)


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
def test_prepared_batch_across_set_window(ctx, oracle, memory):
    """A prepared batch replays one shape; a set_window between executions makes it plan again, and its windows move
    at every execution."""
    rng = np.random.default_rng(6)
    C, bs0, bs1 = 2, 8, 11
    su = make_setup(ctx, C, bs0, bs1, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=[FLOOR])
    S, k, n2 = 4, 3, 1024
    full = [L.PreviousWindowRight(su) for _ in range(S)]
    win = [L.PreviousWindowRight(su) for _ in range(S)]
    modes = np.ones(k, np.uint8)
    stride = (k * n2) + 4
    n_el = S * C * stride
    coeffs = ctx.host_alloc(S * k * C * n2, np.float32)
    fa, wa = Arena(ctx, n_el, F32P, memory, pinned=True), Arena(ctx, n_el, F32P, memory, pinned=True)
    dco = torch.zeros(coeffs.size, dtype=torch.float32, device="cuda") if memory == cabi.MEM_DEVICE else None
    co = dco.data_ptr() if dco is not None else coeffs

    def specs(pw):
        return [L.ChainSpec(pw[i], modes, coeff_offset=i * k * C * n2, packet_index=i * k, out_offset=i * C * stride, out_stride=stride)
                for i in range(S)]
    fb = L.Batch(ctx, specs(full), SPECTRUM, memory, co, fa.ptr, F32P)
    wb = L.Batch(ctx, specs(win), SPECTRUM, memory, co, wa.ptr, F32P)
    pos = 0
    plan = {3: (500, 5000), 5: (0, 1000)}       # execution -> window set on every windowed stream before it
    window = None
    for ex in range(8):
        coeffs[...] = (rng.standard_normal(coeffs.size) * 0.1).astype(np.float32)
        if dco is not None:
            dco.copy_(torch.from_numpy(np.array(coeffs)))
            torch.cuda.synchronize()
        if ex in plan:
            window = plan[ex]
            for w in win:
                w.set_window(*window)
            wpos = pos
        for bt in (fb, wb):
            bt.run()
        ctx.synchronize()
        fbuf, wbuf = fa.read().view(np.float32), wa.read().view(np.float32)
        fr, wr = fb.collect(), wb.collect()
        for i in range(S):
            n = fr[i].n_samples
            if window is None:
                a, e = 0, n
            else:
                s0, lim = window
                a = int(min(max(s0 - (pos - wpos), 0), n))
                e = int(max(a, min(s0 + lim - (pos - wpos), n)))
            assert wr[i].n_samples == e - a, (ex, i, wr[i].n_samples, a, e)
            for c in range(C):
                o = i * C * stride + c * stride
                assert bits_equal(wbuf[o:o + e - a], fbuf[o + a:o + e]), (ex, i, c)
        pos += fr[0].n_samples
    for f, w in zip(full, win):
        assert bits_equal(f.data(), w.data())


def test_single_packet_calls_honour_the_window(ctx, oracle):
    rng = np.random.default_rng(7)
    su = make_setup(ctx, 2, 8, 11, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=[FLOOR])
    a, b = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
    b.set_window(700, 600)
    got_a, got_b = [], []
    for _ in range(4):
        spec = (rng.standard_normal((2, 1024)) * 0.1).astype(np.float32)
        got_a.append(L.decode_spectrum(su, 1, spec, a))
        got_b.append(L.decode_spectrum(su, 1, spec, b))
    full = np.concatenate(got_a, axis=1)
    part = np.concatenate(got_b, axis=1)
    assert bits_equal(part, full[:, 700:1300])
    assert b.window == (0, 0)
    assert bits_equal(a.data(), b.data())
