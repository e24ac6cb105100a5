"""32-bit and packed 24-bit integer PCM (LWB_OUT_I32_* / LWB_OUT_I24_*) on the GPU.

An element is the f32 sample the F32 format of the same layout writes, times 2^31 / 2^23, truncated toward zero and
saturated (NaN -> 0); i24 keeps the low 3 bytes, little-endian.  So the oracle's f32 PCM converted by numpy
(test_int_output_cpu) pins every byte.  Arenas are raw bytes filled with a guard byte, so that every byte outside a
chain's write set -- the bytes on both sides of every 3-byte row included -- can be checked.  Checked:
  1. every store site (k_long, k_long_s, k_mid at both sizes, k_short, k_short_g, k_chain planar, interleaved and with an
     output mix, the four-kernel path with and without a mix) on every edge value of both rules;
  2. whole decodes of the spectrum, residue and VQ entries, planar and interleaved, host and device memory, with
     LWB_FORCE_GENERIC unset, "2" and "1", against the oracle and against the same batch in f32, launching what f32 does;
  3. output windows (odd skips and limits, odd out_offset) on every path: byte-exact, guards untouched (k_row_copy);
  4. asynchronous submits two deep and prepared-batch replays;
  5. the front half: OggStreamReader, skip_samples_linear, OggStreamReaders.read / skip and StreamBatcher.submit;
  6. refusal of formats 6, 7, 12 and -1, with nothing changed."""
import ctypes as ct

import numpy as np
import pytest

import lewton_b200 as L
import vorbis_packer as vp
from helpers import (ALL_KERNELS, FUSED, GENERIC, RefStream, bits_equal, environ, expect_kernels, launches_are_attributed,
                     make_setup, mode_sequence)
from lewton_b200 import _cabi as cabi
from lewton_b200 import api
from lewton_b200 import frontend as fe
from test_frontend_gpu import build_stream, consistent_modes, oracle_pcm, page_granules
from test_int_output_cpu import int_test_values, to_i24, to_i32
from test_vq_shapes_gpu import Batch as PackerBatch
from test_vq_shapes_gpu import Streams

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, F32I = cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED
I32P, I32I, I24P, I24I = cabi.OUT_I32_PLANAR, cabi.OUT_I32_INTERLEAVED, cabi.OUT_I24_PLANAR, cabi.OUT_I24_INTERLEAVED
SPECTRUM, RESIDUE, VQ = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
ESZ = {F32P: 4, F32I: 4, I32P: 4, I32I: 4, I24P: 3, I24I: 3}
F32_OF = {I32P: F32P, I32I: F32I, I24P: F32P, I24I: F32I}
GUARD = 0xA5
MODES = ((0, 0), (1, 0))    # mode 0: short block, mode 1: long block
ALIGN = 16                  # element offsets at which an i24 planar row is 16-byte aligned (the fused kernels' layout)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def planar(fmt):
    return fmt in (F32P, I32P, I24P)


def up(n, a=ALIGN):
    return (n + a - 1) // a * a


def arena(n_elems, fmt, alloc=None):
    """A guard-filled byte arena of n_elems elements of fmt."""
    a = np.empty(n_elems * ESZ[fmt], np.uint8) if alloc is None else alloc((n_elems * ESZ[fmt],), np.uint8)
    a[...] = GUARD
    return a


def elements(raw, fmt):
    """The arena's elements as numbers: int32 for the integer formats, float32 for f32."""
    if fmt in (I24P, I24I):
        return L.i24_to_i32(raw[: raw.size // 3 * 3])
    return raw.view(np.float32 if fmt in (F32P, F32I) else np.int32)


def convert(fmt, f32):
    return (to_i24 if fmt in (I24P, I24I) else to_i32)(f32)


def write_mask(chains, channels, fmt, size):
    """The elements the chains report writing, as a mask over the arena."""
    m = np.zeros(size, bool)
    for c in chains:
        n = int(c.n_samples)
        if planar(fmt):
            for k in range(channels):
                s = int(c.out_offset) + k * int(c.out_stride)
                m[s:s + n] = True
        else:
            m[int(c.out_offset):int(c.out_offset) + n * channels] = True
    return m


def chain_pcm(vals, chain, channels, fmt, n):
    o = int(chain.out_offset)
    if planar(fmt):
        return np.stack([vals[o + k * int(chain.out_stride): o + k * int(chain.out_stride) + n] for k in range(channels)])
    return vals[o:o + n * channels].reshape(n, channels).T


def assert_guard_outside(raw, mask, fmt, what):
    bad = np.nonzero(~np.repeat(mask, ESZ[fmt]) & (raw != GUARD))[0]
    assert not bad.size, f"{what}: {bad.size} bytes outside the write set were written; first at {bad[:4]}"


def assert_ints(got, want, what):
    got, want = np.asarray(got, np.int64), np.asarray(want, np.int64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero(got.ravel() != want.ravel())[0]
    assert not bad.size, (what, f"{bad.size} of {got.size} differ; first at {bad[:4]}: got {got.ravel()[bad[:4]]} "
                                f"want {want.ravel()[bad[:4]]}")


# ---------------------------------------------------------------------------------------------------------------------
# 1: every store site, on every edge value
# ---------------------------------------------------------------------------------------------------------------------
VALUES = int_test_values()

# site: (bs0, bs1, planar, p_short, packets per chain, environment, output mix, kernels that must run, must not)
SITES = {
    "k_long": (8, 11, True, 0.0, 2, None, False, {"k_long"}, ALL_KERNELS - {"k_long"}),
    "k_mid_1024": (10, 10, True, 0.0, 2, None, False, {"k_mid"}, ALL_KERNELS - {"k_mid"}),
    "k_mid_512": (9, 9, True, 0.0, 2, None, False, {"k_mid"}, ALL_KERNELS - {"k_mid"}),
    "k_short": (8, 8, True, 0.0, 4, None, False, {"k_short"}, ALL_KERNELS - {"k_short", "k_row_copy"}),
    "k_long_s_k_short_g": (8, 11, True, 0.3, 12, None, False, {"k_long_s", "k_short_g"}, GENERIC | {"k_long", "k_chain", "k_mid"}),
    "k_long_s_no_bursts": (8, 11, True, 0.3, 12, {"LWB_NO_BURSTS": "1"}, False, {"k_long_s", "k_short"},
                           GENERIC | {"k_long", "k_chain", "k_mid", "k_short_g"}),
    "k_chain_interleaved": (8, 11, False, 0.3, 4, None, False, {"k_chain"}, ALL_KERNELS - {"k_chain"}),
    "k_chain_128_4096": (7, 12, True, 0.3, 4, None, False, {"k_chain"}, ALL_KERNELS - {"k_chain"}),
    "k_chain_mix": (8, 11, False, 0.3, 4, None, True, {"k_chain"}, ALL_KERNELS - {"k_chain"}),
    "k_overlap": (8, 11, True, 0.3, 4, {"LWB_FORCE_GENERIC": "1"}, False, {"k_imdct", "k_overlap", "k_save_state"},
                  FUSED | {"k_chain", "k_prologue"}),
    "k_overlap_mix": (8, 11, False, 0.3, 4, {"LWB_FORCE_GENERIC": "1"}, True, {"k_imdct", "k_overlap", "k_save_state"},
                      FUSED | {"k_chain", "k_prologue"}),
}


@pytest.mark.parametrize("kind", ["i32", "i24"])
@pytest.mark.parametrize("site", list(SITES))
def test_every_store_site_writes_every_edge_value(ctx, site, kind):
    bs0, bs1, is_planar, p_short, P, env, mix, ran, not_ran = SITES[site]
    fmt = {("i32", True): I32P, ("i32", False): I32I, ("i24", True): I24P, ("i24", False): I24I}[(kind, is_planar)]
    Cn = 2
    rng = np.random.default_rng(2400 + len(site))
    tables = []
    for bs in (bs0, bs1):
        t = L.generate_tables(bs)
        t["window"] = np.ones_like(t["window"])            # slopes of 1.0: sample = 0 * 1 + state * 1
        tables.append(t)
    su = make_setup(ctx, Cn, bs0, bs1, modes=MODES, tables=tables)
    if mix:
        su.set_output_mix(L.mix_select(Cn, [1, 0]))         # a permutation: the samples move bit for bit
    n0, n1 = 1 << bs0, 1 << bs1
    chains, wants, pwrs = [], [], []
    at = ooff = coff = 0
    while at < VALUES.size:
        bf, prev, nxt = mode_sequence(rng, P, p_short)
        plen = n1 // 2 if (bf[0] and prev[0]) else n0 // 2
        state = np.zeros((Cn, plen), np.float32)
        take = VALUES[at:at + Cn * plen]
        state.ravel()[:take.size] = take
        at += take.size
        pwr = L.PreviousWindowRight(su)
        pwr.set_data(state)
        n = sum(L.get_decoded_sample_count(su, int(m), bool(p), bool(x)) for m, p, x in zip(bf, prev, nxt))
        want = np.zeros((Cn, n), np.float32)
        want[:, :plen] = state
        if mix:
            want = want[::-1]
        stride = up(n) + ALIGN
        chains.append(L.ChainSpec(pwr, bf, prev, nxt, coeff_offset=coff, out_offset=ooff, out_stride=stride if is_planar else 0))
        coff += sum(Cn * ((n1 if m else n0) // 2) for m in bf)
        ooff += Cn * stride + ALIGN
        wants.append(want)
        pwrs.append(pwr)
    raw = arena(ooff, fmt)
    coeffs = np.zeros(coff, np.float32)
    with environ(env), expect_kernels(ctx, ran=ran, not_ran=not_ran):
        L.decode_chains(ctx, chains, SPECTRUM, HOST, coeffs, raw, fmt)
    vals = elements(raw, fmt)
    for i, (c, w) in enumerate(zip(chains, wants)):
        assert (c.status, c.n_samples) == (0, w.shape[1]), (site, i, c.status, c.n_samples, w.shape)
        assert_ints(chain_pcm(vals, c, Cn, fmt, w.shape[1]), convert(fmt, w), (site, kind, i))
    assert_guard_outside(raw, write_mask(chains, Cn, fmt, ooff), fmt, site)
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: whole decodes, against the oracle and against the same batch in f32
# ---------------------------------------------------------------------------------------------------------------------
class SpectrumCase:
    """S streams of a synthetic setup with random spectra (the last stream's loud enough to saturate), and their
    oracle twins."""

    def __init__(self, ctx, oracle, seed, channels, bs0, bs1, S, n_packets, p_short):
        rng = np.random.default_rng(seed)
        self.C, self.S = channels, S
        self.su = make_setup(ctx, channels, bs0, bs1, modes=MODES)
        self.seqs = [mode_sequence(rng, n_packets, p_short) for _ in range(S)]
        self.specs = [[(rng.standard_normal((channels, (1 << (bs1 if b else bs0)) // 2)) * (30.0 if s == S - 1 else 0.1))
                       .astype(np.float32) for b in self.seqs[s][0]] for s in range(S)]
        self.twins = [RefStream(oracle, channels, bs0, bs1, MODES) for _ in range(S)]

    def advance(self, p0, p1):
        out = []
        for s in range(self.S):
            bf, prev, nxt = self.seqs[s]
            parts = []
            for i in range(p0, p1):
                rc, pcm = self.twins[s].spectrum(int(bf[i]), int(prev[i]), int(nxt[i]), self.specs[s][i])
                assert rc == 0
                parts.append(pcm)
            out.append(np.concatenate(parts, axis=1))
        return out


def relayout(b, C, fmt, skew=0, room=0):
    """Lays batch b's chains out at element offsets and strides that are multiples of 16 (+ skew on every offset), with
    gaps between them and `room` more samples per channel than the oracle's run produced; sets b.n_out."""
    ooff, layout = 0, []
    for (m, p, n, c0, r, _, _), w in zip(b.layout, b.wants):
        stride = up(w.shape[1] + room) + ALIGN
        layout.append((m, p, n, c0, r, ooff + skew, stride if planar(fmt) else 0))
        ooff += C * stride + ALIGN
    b.layout, b.n_out = layout, ooff + skew + ALIGN
    return b


class SpectrumBatch:
    """Packets [p0, p1) of every stream of a SpectrumCase as one spectrum-entry batch."""

    def __init__(self, case, p0, p1, fmt, room=0):
        self.layout, coeffs, coff = [], [], 0
        for s in range(case.S):
            bf, prev, nxt = (a[p0:p1] for a in case.seqs[s])
            self.layout.append((bf.copy(), prev.copy(), nxt.copy(), coff, 0, 0, 0))
            sp = np.concatenate([x.ravel() for x in case.specs[s][p0:p1]])
            coeffs.append(sp)
            coff += sp.size
        self.coeffs = np.concatenate(coeffs)
        self.kinds = self.ys = self.dense = self.vq = None
        self.wants = case.advance(p0, p1)
        relayout(self, case.C, fmt, room=room)

    def chains(self, pwrs):
        return [L.ChainSpec(pwrs[s], m, p, n, coeff_offset=c0, packet_index=r, out_offset=o, out_stride=sd)
                for s, (m, p, n, c0, r, o, sd) in enumerate(self.layout)]


def run_batch(ctx, b, fmt, pwrs, entry, memory, floor_mem=HOST, env=None):
    """One lwb_decode_chains of batch b in fmt over a guard-filled arena: (raw bytes, chains, {kernel: launches})."""
    raw = arena(b.n_out, fmt)
    chains = b.chains(pwrs)
    frees = []

    def dev(a):
        a = np.ascontiguousarray(a)
        p = ctx.device_alloc(max(a.nbytes, 16))
        ctx.h2d(p, a)
        frees.append(p)
        return p

    try:
        kw = {}
        if entry != SPECTRUM:
            kw = dict(floor_kind=b.kinds, floor1_y=b.ys)
            if entry == VQ:
                kw["vq"] = b.vq
            if floor_mem == DEVICE:
                kw = {k: dev(a) if k != "vq" else tuple(dev(x) for x in a) for k, a in kw.items()}
                kw["floor_memory"] = DEVICE
        coeffs = None if entry == VQ else b.coeffs
        dense, out = (b.dense if entry != SPECTRUM else None), raw
        if memory == DEVICE:
            coeffs = None if coeffs is None else dev(coeffs)
            dense = None if dense is None else dev(dense)
            out = dev(raw)
        with environ(env), expect_kernels(ctx) as delta:
            L.decode_chains(ctx, chains, entry, memory, coeffs, out, fmt, dense_floor=dense, **kw)
        ctx.synchronize()
        if memory == DEVICE:
            ctx.d2h(raw, out)
    finally:
        for p in frees:
            ctx.device_free(p)
    return raw, chains, {k: v for k, v in delta.items() if v}


def check_formats(ctx, batches, make_pwrs, C, fmt, entry, memory, floor_mem=HOST, env=None, twins=None):
    """Runs `batches` in order in fmt and in its f32 sibling (fresh streams each) and checks the integer runs."""
    f32 = F32_OF[fmt]
    runs, states = {}, {}
    for f in (f32, fmt):
        pwrs = make_pwrs()
        runs[f] = [run_batch(ctx, b, f, pwrs, entry, memory, floor_mem, env) for b in batches]
        states[f] = [p.data() for p in pwrs]
        for p in pwrs:
            p.close()
    for k, b in enumerate(batches):
        raw, chains, ran = runs[fmt][k]
        raw32, _, ran32 = runs[f32][k]
        what = (fmt, entry, memory, env, k)
        assert ran == ran32, (what, "launched", ran, "f32 launched", ran32)
        vals, vals32 = elements(raw, fmt), elements(raw32, f32)
        for s, (w, c) in enumerate(zip(b.wants, chains)):
            assert (c.status, c.n_samples) == (0, w.shape[1]), (what, s, c.status, c.n_samples, w.shape)
            assert_ints(chain_pcm(vals, c, C, fmt, w.shape[1]), convert(fmt, w), (what, s, "oracle"))
        mask = write_mask(chains, C, fmt, b.n_out)
        assert_ints(vals[mask], convert(fmt, vals32[mask]), (what, "the f32 arena converted"))
        assert_guard_outside(raw, mask, fmt, what)
    for s, (a, b) in enumerate(zip(states[fmt], states[f32])):
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), ("end state", s)
        if twins is not None:
            w = twins[s].pwr.data()
            assert (a is None) == (w is None) and (a is None or bits_equal(a, w)), ("end state vs oracle", s)


ENVS = [None, {"LWB_FORCE_GENERIC": "2"}, {"LWB_FORCE_GENERIC": "1"}]


# channels, bs0, bs1, memory, p_short
SPECTRUM_CASES = [
    (2, 8, 11, HOST, 0.0),           # k_long
    (2, 8, 11, DEVICE, 0.3),         # mixed: k_long_s + bursts
    (2, 8, 8, HOST, 0.0),            # k_short
    (6, 9, 9, DEVICE, 0.0),          # k_mid
    (2, 6, 13, HOST, 0.3),           # 64/8192: k_chain
]


@pytest.mark.parametrize("fmt", [I32P, I24P, I32I, I24I])
@pytest.mark.parametrize("env", ENVS, ids=["paths", "chain", "four_kernel"])
@pytest.mark.parametrize("channels,bs0,bs1,memory,p_short", SPECTRUM_CASES)
def test_spectrum_batches_match_the_oracle_and_f32(ctx, oracle, channels, bs0, bs1, memory, p_short, env, fmt):
    S, P, K = 3, 4, 2
    case = SpectrumCase(ctx, oracle, 2500 + 31 * channels + bs0 + 3 * bs1 + fmt, channels, bs0, bs1, S, P * K, p_short)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, fmt) for k in range(K)]
    check_formats(ctx, batches, lambda: [L.PreviousWindowRight(case.su) for _ in range(S)], channels, fmt, SPECTRUM, memory,
                  env=env, twins=case.twins)


# channels, bs0, bs1, residue type, floor-0 records, memory, floor / VQ memory, entry, p_short
PACKER_CASES = [
    (2, 8, 11, 1, False, DEVICE, HOST, VQ, 0.0),
    (2, 8, 11, 2, True, HOST, HOST, RESIDUE, 0.0),
    (2, 8, 11, None, False, HOST, DEVICE, RESIDUE, 0.3),
    (6, 10, 10, 0, False, DEVICE, DEVICE, VQ, 0.3),
    (2, 9, 9, 2, True, HOST, HOST, VQ, 0.3),
    (1, 7, 12, 1, True, HOST, DEVICE, VQ, 0.3),
]


@pytest.mark.parametrize("fmt", [I32P, I24P, I24I])
@pytest.mark.parametrize("env", ENVS, ids=["paths", "chain", "four_kernel"])
@pytest.mark.parametrize("channels,bs0,bs1,rtype,records,memory,floor_mem,entry,p_short", PACKER_CASES)
def test_packer_streams_match_the_oracle_and_f32(ctx, oracle, channels, bs0, bs1, rtype, records, memory, floor_mem, entry,
                                                 p_short, env, fmt):
    S, P, K = 3, 4, 2
    seed = 24000 + 97 * channels + 13 * bs0 + bs1 + (7 if records else 0)
    st = Streams(seed, channels, bs0, bs1, rtype, records, S, P * K, p_short=p_short)
    su = st.hdr.make_setup(ctx, floor0=records)
    twins = st.twins(oracle)
    batches = [relayout(PackerBatch(st, k * P, (k + 1) * P, cabi.OUT_I16_PLANAR if planar(fmt) else cabi.OUT_I16_INTERLEAVED,
                                    twins), channels, fmt) for k in range(K)]
    check_formats(ctx, batches, lambda: [L.PreviousWindowRight(su) for _ in range(S)], channels, fmt, entry, memory, floor_mem,
                  env, twins)


# ---------------------------------------------------------------------------------------------------------------------
# 3: output windows: odd skips, odd limits, odd out_offset, byte-exact with guards on both sides of every row
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [I24P, I24I, I32P])
@pytest.mark.parametrize("skew", [0, 1, 5])
@pytest.mark.parametrize("env", ENVS, ids=["paths", "chain", "four_kernel"])
@pytest.mark.parametrize("memory", [HOST, DEVICE])
def test_output_windows_are_byte_exact(ctx, oracle, fmt, skew, env, memory):
    S, P, C = 4, 6, 2
    case = SpectrumCase(ctx, oracle, 2600 + fmt + skew, C, 8, 11, S, P, 0.0)
    b = relayout(SpectrumBatch(case, 0, P, fmt), C, fmt, skew)
    windows = [(3, 1001), (0, 7), (1023, None), (5, 0)]
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    for p, (sk, lim) in zip(pwrs, windows):
        p.set_window(sk, lim)
    raw, chains, ran = run_batch(ctx, b, fmt, pwrs, SPECTRUM, memory, env=env)
    if skew == 0 and env is None and planar(fmt):
        assert ran.get("k_long") and ran.get("k_row_copy"), ran          # the fused path, then the row copies
    vals = elements(raw, fmt)
    for s, (w, c, (sk, lim)) in enumerate(zip(b.wants, chains, windows)):
        want = w[:, sk: None if lim is None else sk + lim]
        assert (c.status, c.n_samples) == (0, want.shape[1]), (s, c.status, c.n_samples, want.shape)
        assert_ints(chain_pcm(vals, c, C, fmt, want.shape[1]), convert(fmt, want), (fmt, skew, env, memory, s))
    assert_guard_outside(raw, write_mask(chains, C, fmt, b.n_out), fmt, (fmt, skew, env, memory))
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: asynchronous and prepared batches
# ---------------------------------------------------------------------------------------------------------------------
def _check_oracle(raw, chains, wants, C, fmt, n_out, what):
    vals = elements(raw, fmt)
    for s, (w, c) in enumerate(zip(wants, chains)):
        assert (c.status, c.n_samples) == (0, w.shape[1]), (what, s, c.status, c.n_samples)
        assert_ints(chain_pcm(vals, c, C, fmt, w.shape[1]), convert(fmt, w), (what, s))
    assert_guard_outside(raw, write_mask(chains, C, fmt, n_out), fmt, what)


@pytest.mark.parametrize("fmt", [I32P, I24P, I32I, I24I])
def test_submits_two_deep(ctx, oracle, fmt):
    S, P, C = 6, 6, 2
    case = SpectrumCase(ctx, oracle, 2700 + fmt, C, 8, 11, S, 2 * P, 0.3)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, fmt) for k in range(2)]
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    tickets, arenas = [], []
    for b in batches:
        coeffs = ctx.host_alloc(b.coeffs.shape, np.float32)
        coeffs[...] = b.coeffs
        raw = arena(b.n_out, fmt, ctx.host_alloc)
        arenas.append(raw)
        tickets.append(ctx.submit_chains(b.chains(pwrs), SPECTRUM, HOST, coeffs, raw, fmt))
    for k, (t, b, raw) in enumerate(zip(tickets, batches, arenas)):
        _check_oracle(raw, t.wait(), b.wants, C, fmt, b.n_out, ("submit", k))
    for p, tw in zip(pwrs, case.twins):
        assert bits_equal(p.data(), tw.pwr.data())
        p.close()


@pytest.mark.parametrize("fmt", [I32P, I24P])
def test_prepared_batch_replays_and_replans(ctx, oracle, fmt):
    S, P, C = 8, 4, 2
    case = SpectrumCase(ctx, oracle, 2800 + fmt, C, 8, 11, S, P, 0.0)
    b = SpectrumBatch(case, 0, P, fmt, room=1024)           # (replays with state emit the first packet's 1024 samples too)
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    raw = arena(b.n_out, fmt)
    plan = L.Batch(ctx, b.chains(pwrs), SPECTRUM, HOST, b.coeffs, raw, fmt)
    wants = b.wants
    for step in range(5):
        if step == 3:
            for p, tw in zip(pwrs, case.twins):
                p.reset()
                tw.pwr.reset()
        if step:
            wants = case.advance(0, P)
        raw[...] = GUARD
        with expect_kernels(ctx, ran={"k_long"}, not_ran=ALL_KERNELS - {"k_long"}):
            plan.run()
        _check_oracle(raw, plan.collect(), wants, C, fmt, b.n_out, ("step", step))
    for p, tw in zip(pwrs, case.twins):
        assert bits_equal(p.data(), tw.pwr.data())
    plan.close()
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: the front half, against f32 from the same calls
# ---------------------------------------------------------------------------------------------------------------------
def widen(a, kind):
    a = np.asarray(a)
    return L.i24_to_i32(a) if kind == "i24" else a.astype(np.int64)


@pytest.mark.parametrize("kind", ["i32", "i24"])
@pytest.mark.parametrize("seed,channels,floor0", [(2401, 2, False), (2402, 6, True)])
def test_ogg_stream_reader(ctx, oracle, seed, channels, floor0, kind):
    spec, packets, infos = build_stream(seed, channels, floor0, 14)
    want, _ = oracle_pcm(oracle, spec, infos)
    cut = 37
    data = vp.ogg_stream(0x2424, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets,
                         page_granules(want, 3, cut), packets_per_page=3)
    for interleaved in (False, True):
        rd, rf = fe.OggStreamReader(ctx, data), fe.OggStreamReader(ctx, data)
        for i, w in enumerate(want):
            n = w.shape[1] - (cut if i == len(want) - 1 else 0)
            got = rd.read_dec_packet_generic(kind, interleaved)
            f32 = rf.read_dec_packet_generic("f32", interleaved)
            got = widen(got, kind).reshape(n, channels).T if interleaved else np.stack([widen(g, kind) for g in got])
            f32 = np.asarray(f32).reshape(n, channels).T if interleaved else np.stack(f32)
            assert_ints(got, convert(I24P if kind == "i24" else I32P, w[:, :n]), (interleaved, i, "oracle"))
            assert_ints(got, convert(I24P if kind == "i24" else I32P, f32), (interleaved, i, "f32"))
        assert rd.read_dec_packet_generic(kind, interleaved) is None
        rd.close()
        rf.close()


@pytest.mark.parametrize("kind", ["i32", "i24"])
def test_skip_samples_linear(ctx, oracle, kind):
    n_packets, per_page, channels = 17, 3, 2
    spec, packets, infos = build_stream(2410, channels, False, n_packets)
    want, _ = oracle_pcm(oracle, spec, infos)
    gran = page_granules(want, per_page, 11)
    data = vp.ogg_stream(0x2425, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets, gran,
                         packets_per_page=per_page)
    rd, rf = fe.OggStreamReader(ctx, data), fe.OggStreamReader(ctx, data)
    fmt = I24P if kind == "i24" else I32P
    rd.read_dec_packet_generic(kind)
    rf.read_dec_packet_generic("f32")
    for to_skip in (3, 2500, 41, 10 ** 7):
        got, left = rd.skip_samples_linear(to_skip, sample=kind)
        f32, fleft = rf.skip_samples_linear(to_skip, sample="f32")
        assert left == fleft, (to_skip, left, fleft)
        if f32 is None:
            assert got is None
            continue
        assert_ints(np.stack([widen(g, kind) for g in got]), convert(fmt, np.stack(f32)), to_skip)
    rd.close()
    rf.close()


def _streams(ctx, oracle, seed, n, channels=2):
    out = []
    for k in range(n):
        spec, packets, infos = build_stream(seed + k, channels, False, 9)
        want, _ = oracle_pcm(oracle, spec, infos)
        out.append(vp.ogg_stream(0x2500 + k, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets,
                                 page_granules(want, 3, 0), packets_per_page=3))
    return out


@pytest.mark.parametrize("kind", ["i32", "i24"])
def test_ogg_stream_readers_read_and_skip(ctx, oracle, kind):
    datas = _streams(ctx, oracle, 2420, 3)
    fmt = I24P if kind == "i24" else I32P
    got_rs, f32_rs = fe.OggStreamReaders(ctx), fe.OggStreamReaders(ctx)
    for d in datas:
        got_rs.add(d)
        f32_rs.add(d)
    for step in range(3):
        got = got_rs.read_dec_packets(range(3), 2, sample=kind)
        f32 = f32_rs.read_dec_packets(range(3), 2, sample="f32")
        assert len(got) == len(f32)
        for g, f in zip(got, f32):
            assert len(g) == len(f)
            for gp, fp in zip(g, f):
                if isinstance(fp, list):
                    assert_ints(np.stack([widen(x, kind) for x in gp]), convert(fmt, np.stack(fp)), (step,))
                else:
                    assert type(gp) is type(fp), (gp, fp)
        g = got_rs.skip_samples_linear_dec(range(3), [700, 3, 5000], sample=kind)
        f = f32_rs.skip_samples_linear_dec(range(3), [700, 3, 5000], sample="f32")
        for (gp, gl), (fp, fl) in zip(g, f):
            assert gl == fl and (gp is None) == (fp is None)
            if fp is not None:
                assert_ints(np.stack([widen(x, kind) for x in gp]), convert(fmt, np.stack(fp)), ("skip", step))
    got_rs.close()
    f32_rs.close()


@pytest.mark.parametrize("fmt", [I32P, I24P])
@pytest.mark.parametrize("memory", [HOST, DEVICE])
def test_stream_batcher_submit(ctx, oracle, fmt, memory):
    import torch
    channels, P, S = 2, 8, 6
    rng = np.random.default_rng(2430)
    spec = vp.StreamSpec(rng, channels=channels)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    pkts = [spec.audio_packet(m, p, n)[0] for m, p, n in consistent_modes(spec, rng, P, p_short=0.2)]
    stride = up(P * (1 << spec.bs1) // 2)
    out = {}
    for f in (F32_OF[fmt], fmt):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        nbytes = S * channels * stride * ESZ[f]
        if memory == DEVICE:
            pcm = torch.full((nbytes,), GUARD, dtype=torch.uint8, device="cuda")
        else:
            pcm = arena(S * channels * stride, f, ctx.host_alloc)
        bt = fe.StreamBatcher(ctx, hdr, threads=2)
        res = bt.submit([(pwrs[s], list(pkts)) for s in range(S)], pcm, stride, out_format=f).wait()
        bt.close()
        raw = pcm.cpu().numpy() if memory == DEVICE else np.array(pcm)
        out[f] = (res, raw)
        for p in pwrs:
            p.close()
    (res32, raw32), (res, raw) = out[F32_OF[fmt]], out[fmt]
    assert [tuple(r) for r in res] == [tuple(r) for r in res32]
    vals, vals32 = elements(raw, fmt), elements(raw32, F32_OF[fmt])
    mask = np.zeros(S * channels * stride, bool)
    for s in range(S):
        n = tuple(res32[s])[0]
        for k in range(channels):
            mask[(s * channels + k) * stride:(s * channels + k) * stride + n] = True
    assert mask.any()
    assert_ints(vals[mask], convert(fmt, vals32[mask]), "batcher")
    assert_guard_outside(raw, mask, fmt, "batcher")


# ---------------------------------------------------------------------------------------------------------------------
# 6: formats that are not assigned are refused, with nothing changed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [6, 7, 12, -1])
def test_unassigned_formats_are_refused_untouched(ctx, oracle, bad):
    S, P, Cn = 2, 3, 2
    case = SpectrumCase(ctx, oracle, 2900, Cn, 8, 11, S, 2 * P, 0.0)
    b0, b1 = SpectrumBatch(case, 0, P, I32P), SpectrumBatch(case, P, 2 * P, I32P)
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    run_batch(ctx, b0, I32P, pwrs, SPECTRUM, HOST)
    states = [p.data() for p in pwrs]
    lib = cabi.lib()
    raw = arena(b1.n_out, I32P)
    arr, io = api._marshal(b1.chains(pwrs), SPECTRUM, HOST, b1.coeffs, raw, bad, None, None, None, HOST, None)
    for i in range(S):
        arr[i].n_samples, arr[i].packets_done, arr[i].status = 1234, 56, -7

    def untouched(what):
        for i in range(S):
            assert (arr[i].n_samples, arr[i].packets_done, arr[i].status) == (1234, 56, -7), (what, i)
        for p, s in zip(pwrs, states):
            assert bits_equal(p.data(), s), what
        assert (raw == GUARD).all(), what

    with expect_kernels(ctx, ran={}, not_ran=ALL_KERNELS):
        assert lib.lwb_decode_chains(ctx._h, arr, S, ct.byref(io)) == cabi.ERR_INVALID
        assert lib.lwb_last_error(ctx._h).decode() == "bad out_format"
        untouched("decode_chains")
        t = ct.c_uint64()
        assert lib.lwb_submit_chains(ctx._h, arr, S, ct.byref(io), ct.byref(t)) == cabi.ERR_INVALID
        untouched("submit_chains")
        plan = ct.c_void_p()
        assert lib.lwb_plan_create(ctx._h, arr, S, ct.byref(io), ct.byref(plan)) == 0
        assert lib.lwb_plan_execute(plan) == cabi.ERR_INVALID
        lib.lwb_plan_destroy(plan)
        untouched("plan_execute")
        n = ct.c_size_t()
        spec = np.zeros((Cn, 1024), np.float32)
        out = np.full(Cn * 2048 * 4, GUARD, np.uint8)
        assert lib.lwb_decode_spectrum(pwrs[0]._h, 1, 1, 1, spec.ctypes.data, bad, out.ctypes.data, 2048,
                                       ct.byref(n)) == cabi.ERR_INVALID
        assert (out == GUARD).all()
        untouched("decode_spectrum")
    for p in pwrs:
        p.close()
