"""Half-precision PCM (LWB_OUT_F16_PLANAR / LWB_OUT_F16_INTERLEAVED) on the GPU.

An f16 element is the IEEE round-to-nearest-even binary16 of the f32 sample the F32 format of the same layout writes, so
the oracle's f32 PCM converted by numpy pins it bit for bit (up to the sign of zero; any NaN equals any NaN).  Checked:
  1. every store site (k_long, k_mid at both sizes, k_short, the one-pass mixed schedule with and without bursts, k_chain
     planar and interleaved, the four-kernel path) on every f32 -> f16 rounding boundary: window slopes of 1.0 and a
     zero spectrum make a packet's first samples exactly the f32 values imported as its stream state;
  2. whole decodes of the spectrum, residue and VQ entries against the oracle, and against the same batch in f32 and in
     i16: the f16 arena is the f32 arena converted, nothing outside the write set changes, the end states are the f32
     run's, and the kernels launched are exactly the i16 run's (f16 takes i16's paths);
  3. asynchronous submits and prepared batches (replays, a re-plan after a reset);
  4. the front half: OggStreamReader.read_dec_packet_generic / skip_samples_linear and lwf_batcher;
  5. refusal of formats past the last one, with nothing changed."""
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
from test_f16_output_cpu import f16_test_values, to_f16
from test_frontend_gpu import _ReaderModel, build_stream, consistent_modes, oracle_pcm, page_granules
from test_vq_shapes_gpu import Batch as PackerBatch
from test_vq_shapes_gpu import Streams

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED
F16P, F16I = cabi.OUT_F16_PLANAR, cabi.OUT_F16_INTERLEAVED
SPECTRUM, RESIDUE, VQ = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
SIBLINGS = {F16P: (F32P, I16P), F16I: (F32I, I16I)}        # the f32 and i16 formats of an f16 format's layout
DTYPES = {F32P: np.float32, F32I: np.float32, I16P: np.int16, I16I: np.int16, F16P: np.float16, F16I: np.float16}
F16_GUARD = 0x7d5a          # a signalling f16 NaN with a fixed payload: the conversion only ever writes quiet NaNs
GUARDS = {np.dtype(np.float32): (np.uint32, 0x7fa5a5a5), np.dtype(np.int16): (np.uint16, 0x5a5a),
          np.dtype(np.float16): (np.uint16, F16_GUARD)}
MODES = ((0, 0), (1, 0))    # mode 0: short block, mode 1: long block


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def planar(fmt):
    return fmt in (F32P, I16P, F16P)


def fill(a):
    """The arena's sentinel in every element; returns the arena."""
    u, g = GUARDS[a.dtype]
    a.view(u)[...] = g
    return a


def same_f16(got, want):
    """Bit-identical float16 arrays up to the sign of zero; any NaN equals any NaN."""
    got, want = np.asarray(got, np.float16), np.asarray(want, np.float16)
    if got.shape != want.shape:
        return False
    return bool(np.all((got.view(np.uint16) == want.view(np.uint16)) | ((got == 0) & (want == 0)) |
                       (np.isnan(got) & np.isnan(want))))


def report(got, want):
    got, want = np.asarray(got, np.float16).ravel(), np.asarray(want, np.float16).ravel()
    bad = np.nonzero(~((got.view(np.uint16) == want.view(np.uint16)) | ((got == 0) & (want == 0)) |
                       (np.isnan(got) & np.isnan(want))))[0]
    return (f"{bad.size} of {got.size} differ; first at {bad[:4]}: got {got.view(np.uint16)[bad[:4]]} "
            f"want {want.view(np.uint16)[bad[:4]]}")


def write_mask(chains, channels, fmt, size):
    """The elements the chains report writing (include/lewton_b200.h, lwb_chain), as a mask over the arena."""
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


def chain_pcm(pcm, chain, channels, fmt, n):
    """[channels][n] of one chain's output."""
    o = int(chain.out_offset)
    if planar(fmt):
        return np.stack([pcm[o + k * int(chain.out_stride): o + k * int(chain.out_stride) + n] for k in range(channels)])
    return pcm[o:o + n * channels].reshape(n, channels).T


def assert_guard_outside(pcm, mask, what):
    u, g = GUARDS[pcm.dtype]
    bad = np.nonzero(~mask & (pcm.view(u) != g))[0]
    assert not bad.size, f"{what}: {bad.size} elements outside the write set were written; first at {bad[:4]}"


# ---------------------------------------------------------------------------------------------------------------------
# 1: every store site, on every rounding boundary
# ---------------------------------------------------------------------------------------------------------------------
VALUES = f16_test_values()

# site: (bs0, bs1, format, p_short, packets per chain, environment, kernels that must run, kernels that must not)
SITES = {
    "k_long": (8, 11, F16P, 0.0, 2, None, {"k_long"}, ALL_KERNELS - {"k_long"}),
    "k_mid_1024": (10, 10, F16P, 0.0, 2, None, {"k_mid"}, ALL_KERNELS - {"k_mid"}),
    "k_mid_512": (9, 9, F16P, 0.0, 2, None, {"k_mid"}, ALL_KERNELS - {"k_mid"}),
    "k_short": (8, 8, F16P, 0.0, 4, None, {"k_short"}, ALL_KERNELS - {"k_short", "k_row_copy"}),
    "one_pass": (8, 11, F16P, 0.3, 12, None, {"k_long_s", "k_short_g"}, GENERIC | {"k_long", "k_chain", "k_mid"}),
    "one_pass_no_bursts": (8, 11, F16P, 0.3, 12, {"LWB_NO_BURSTS": "1"}, {"k_long_s", "k_short"},
                           GENERIC | {"k_long", "k_chain", "k_mid", "k_short_g"}),
    "k_chain_interleaved": (8, 11, F16I, 0.3, 4, None, {"k_chain"}, ALL_KERNELS - {"k_chain"}),
    "k_chain_128_4096": (7, 12, F16P, 0.3, 4, None, {"k_chain"}, ALL_KERNELS - {"k_chain"}),
    "four_kernel": (8, 11, F16P, 0.3, 4, {"LWB_FORCE_GENERIC": "1"}, {"k_imdct", "k_overlap", "k_save_state"},
                    FUSED | {"k_chain", "k_prologue"}),
}


@pytest.mark.parametrize("site", list(SITES))
def test_every_store_site_rounds_like_numpy(ctx, site):
    bs0, bs1, fmt, p_short, P, env, ran, not_ran = SITES[site]
    Cn = 2
    rng = np.random.default_rng(1600 + len(site))
    tables = []
    for bs in (bs0, bs1):
        t = L.generate_tables(bs)
        t["window"] = np.ones_like(t["window"])            # slopes of 1.0: sample = 0 * 1 + state * 1
        tables.append(t)
    su = make_setup(ctx, Cn, bs0, bs1, modes=MODES, tables=tables)
    n0, n1 = 1 << bs0, 1 << bs1
    chains, wants, pwrs = [], [], []
    at = ooff = coff = 0
    while at < VALUES.size:
        bf, prev, nxt = mode_sequence(rng, P, p_short)
        # the right half the first packet overlaps with: a long one only ahead of a long block with a long neighbour
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
        stride = (n + 3) // 4 * 4 + 4
        chains.append(L.ChainSpec(pwr, bf, prev, nxt, coeff_offset=coff, out_offset=ooff,
                                  out_stride=stride if planar(fmt) else 0))
        coff += sum(Cn * ((n1 if m else n0) // 2) for m in bf)
        ooff += Cn * stride + 4
        wants.append(want)
        pwrs.append(pwr)
    pcm = fill(np.empty(ooff, np.float16))
    coeffs = np.zeros(coff, np.float32)
    with environ(env), expect_kernels(ctx, ran=ran, not_ran=not_ran):
        L.decode_chains(ctx, chains, SPECTRUM, HOST, coeffs, pcm, fmt)
    for i, (c, w) in enumerate(zip(chains, wants)):
        assert (c.status, c.n_samples) == (0, w.shape[1]), (site, i, c.status, c.n_samples, w.shape)
        got = chain_pcm(pcm, c, Cn, fmt, w.shape[1])
        assert same_f16(got, to_f16(w)), (site, i, report(got, to_f16(w)))
    assert_guard_outside(pcm, write_mask(chains, Cn, fmt, pcm.size), site)
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: whole decodes, against the oracle and against the same batch in f32 and i16
# ---------------------------------------------------------------------------------------------------------------------
class SpectrumCase:
    """S streams of a synthetic setup with random spectra (the last stream's scaled so that its PCM overflows f16), and
    their oracle twins."""

    def __init__(self, ctx, oracle, seed, channels, bs0, bs1, S, n_packets, p_short, loud=True):
        rng = np.random.default_rng(seed)
        self.C, self.S, self.bs0, self.bs1 = channels, S, bs0, bs1
        self.su = make_setup(ctx, channels, bs0, bs1, modes=MODES)
        self.seqs = [mode_sequence(rng, n_packets, p_short) for _ in range(S)]
        self.specs = []
        for s in range(S):
            scale = 3e5 if loud and s == S - 1 else 0.1
            self.specs.append([(rng.standard_normal((channels, (1 << (bs1 if b else bs0)) // 2)) * scale).astype(np.float32)
                               for b in self.seqs[s][0]])
        self.twins = [RefStream(oracle, channels, bs0, bs1, MODES) for _ in range(S)]

    def advance(self, p0, p1):
        """The oracle's PCM of packets [p0, p1) of every stream, twins advanced over them."""
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


class SpectrumBatch:
    """Packets [p0, p1) of every stream of a SpectrumCase as one spectrum-entry batch, laid out like PackerBatch."""

    def __init__(self, case, p0, p1, fmt):
        self.C, self.fmt = case.C, fmt
        self.layout, coeffs = [], []
        coff = ooff = 0
        for s in range(case.S):
            bf, prev, nxt = (a[p0:p1] for a in case.seqs[s])
            n = sum(L.get_decoded_sample_count(case.su, int(m), bool(p), bool(x)) for m, p, x in zip(bf, prev, nxt))
            stride = (n + 3) // 4 * 4 + 4
            self.layout.append((bf.copy(), prev.copy(), nxt.copy(), coff, 0, ooff, stride if planar(fmt) else 0))
            sp = np.concatenate([x.ravel() for x in case.specs[s][p0:p1]])
            coeffs.append(sp)
            coff += sp.size
            ooff += case.C * stride + 4
        self.coeffs, self.n_out = np.concatenate(coeffs), ooff
        self.kinds = self.ys = self.dense = self.vq = None
        self.wants = case.advance(p0, p1)

    def chains(self, pwrs):
        return [L.ChainSpec(pwrs[s], m, p, n, coeff_offset=c0, packet_index=r, out_offset=o, out_stride=sd)
                for s, (m, p, n, c0, r, o, sd) in enumerate(self.layout)]


def run_batch(ctx, b, fmt, pwrs, entry, memory, floor_mem=HOST, env=None):
    """One lwb_decode_chains of batch b (PackerBatch or SpectrumBatch) in `fmt` over a sentinel-filled arena:
    (pcm, chains, {kernel: launches})."""
    pcm = fill(np.empty(b.n_out, DTYPES[fmt]))
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
        dense, out = (b.dense if entry != SPECTRUM else None), pcm
        if memory == DEVICE:
            coeffs = None if coeffs is None else dev(coeffs)
            dense = None if dense is None else dev(dense)
            out = dev(pcm)
        with environ(env), expect_kernels(ctx) as delta:
            L.decode_chains(ctx, chains, entry, memory, coeffs, out, fmt, dense_floor=dense, **kw)
        ctx.synchronize()
        if memory == DEVICE:
            ctx.d2h(pcm, out)
    finally:
        for p in frees:
            ctx.device_free(p)
    return pcm, chains, {k: v for k, v in delta.items() if v}


def check_formats(ctx, batches, make_pwrs, C, fmt, entry, memory, floor_mem=HOST, env=None, key=None, twins=None):
    """Runs `batches` in order in fmt and in its f32 and i16 siblings (fresh streams each) and checks the f16 runs."""
    f32, i16 = SIBLINGS[fmt]
    runs, states = {}, {}
    for f in (f32, i16, fmt):
        pwrs = make_pwrs()
        runs[f] = [run_batch(ctx, b, f, pwrs, entry, memory, floor_mem, env) for b in batches]
        states[f] = [p.data() for p in pwrs]
        for p in pwrs:
            p.close()
    for k, b in enumerate(batches):
        pcm16, chains, ran16 = runs[fmt][k]
        pcm32, _, _ = runs[f32][k]
        what = (fmt, entry, memory, k)
        assert ran16 == runs[i16][k][2], (what, "f16 launched", ran16, "i16 launched", runs[i16][k][2])
        if key is not None:
            want_key = key(b) if callable(key) else key
            assert any(ran16.get(x) for x in want_key), (what, "expected one of", want_key, "launched", ran16)
        for s, (w, c) in enumerate(zip(b.wants, chains)):
            assert (c.status, c.n_samples) == (0, w.shape[1]), (what, s, c.status, c.n_samples, w.shape)
            got = chain_pcm(pcm16, c, C, fmt, w.shape[1])
            assert same_f16(got, to_f16(w)), (what, s, report(got, to_f16(w)))
        mask = write_mask(chains, C, fmt, pcm16.size)
        assert same_f16(pcm16[mask], to_f16(pcm32[mask])), (what, "f16 arena != f32 arena converted")
        assert_guard_outside(pcm16, mask, what)
    for s, (a, b) in enumerate(zip(states[fmt], states[f32])):
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), ("end state", s)
        if twins is not None:
            w = twins[s].pwr.data()
            assert (a is None) == (w is None) and (a is None or bits_equal(a, w)), ("end state vs oracle", s)


MID_OR_CHAIN = lambda b: ("k_mid",) if b.uniform else ("k_chain",)          # noqa: E731
ANY_FUSED = tuple(sorted(FUSED))

# channels, bs0, bs1, residue type, floor-0 records, f16 format, memory, floor / VQ memory, entry, p_short, kernels (one
# of which must run), environment
PACKER_CASES = [
    (2, 8, 11, 1, False, F16P, DEVICE, HOST, VQ, 0.0, ("k_long",), None),             # uniform long
    (2, 8, 11, 2, True, F16P, HOST, HOST, RESIDUE, 0.0, ("k_long",), None),
    (2, 8, 11, None, False, F16P, HOST, DEVICE, RESIDUE, 0.3, ANY_FUSED, None),       # 256/2048 mixed
    (6, 10, 10, 0, False, F16P, DEVICE, DEVICE, VQ, 0.3, MID_OR_CHAIN, None),         # uniform 1024
    (2, 9, 9, 2, True, F16P, HOST, HOST, VQ, 0.3, MID_OR_CHAIN, None),                # uniform 512
    (8, 10, 10, 1, False, F16I, HOST, HOST, RESIDUE, 0.3, ("k_chain",), None),        # interleaved
    (1, 7, 12, 1, True, F16P, HOST, DEVICE, VQ, 0.3, ("k_chain",), None),             # 128/4096
    (2, 6, 13, None, False, F16I, DEVICE, HOST, RESIDUE, 0.3, ("k_chain",), None),    # 64/8192
    (6, 8, 11, 2, True, F16I, HOST, HOST, VQ, 0.2, ("k_chain",), None),
    (2, 8, 11, 1, False, F16P, HOST, HOST, RESIDUE, 0.3, ("k_imdct",), {"LWB_FORCE_GENERIC": "1"}),   # four-kernel path
]


@pytest.mark.parametrize("channels,bs0,bs1,rtype,records,fmt,memory,floor_mem,entry,p_short,key,env", PACKER_CASES)
def test_packer_streams_match_the_oracle_and_f32(ctx, oracle, channels, bs0, bs1, rtype, records, fmt, memory, floor_mem,
                                                 entry, p_short, key, env):
    """Residue and VQ entries of packer bitstreams (floor 1, floor-0 records, unused floors), two batches that carry state."""
    S, P, K = 3, 4, 2
    seed = 16000 + 97 * channels + 13 * bs0 + bs1 + 5 * fmt + (7 if records else 0)
    st = Streams(seed, channels, bs0, bs1, rtype, records, S, P * K, p_short=p_short)
    su = st.hdr.make_setup(ctx, floor0=records)
    twins = st.twins(oracle)
    layout_fmt = I16P if planar(fmt) else I16I               # (PackerBatch lays out planar or interleaved by format)
    batches = [PackerBatch(st, k * P, (k + 1) * P, layout_fmt, twins) for k in range(K)]
    check_formats(ctx, batches, lambda: [L.PreviousWindowRight(su) for _ in range(S)], channels, fmt, entry, memory, floor_mem,
                  env, key, twins)


# channels, bs0, bs1, f16 format, memory, p_short, kernels (one of which must run)
SPECTRUM_CASES = [
    (2, 8, 8, F16P, HOST, 0.0, ("k_short",)),               # 256/256
    (2, 8, 11, F16P, DEVICE, 0.3, ANY_FUSED),               # 256/2048 with bursts
    (1, 8, 11, F16P, HOST, 0.0, ("k_long",)),
    (6, 9, 9, F16P, DEVICE, 0.0, ("k_mid",)),
    (10, 8, 11, F16P, HOST, 0.3, ("k_imdct",)),             # more than 8 channels: the four-kernel path
    (10, 8, 11, F16I, DEVICE, 0.3, ("k_imdct",)),
    (2, 6, 13, F16I, HOST, 0.3, ("k_chain",)),             # 64/8192
    (8, 6, 13, F16P, HOST, 0.3, ("k_imdct",)),              # 8 x 8192: beyond k_chain's shared memory
]


@pytest.mark.parametrize("channels,bs0,bs1,fmt,memory,p_short,key", SPECTRUM_CASES)
def test_spectrum_batches_match_the_oracle_and_f32(ctx, oracle, channels, bs0, bs1, fmt, memory, p_short, key):
    S, P, K = 4, 5, 2
    case = SpectrumCase(ctx, oracle, 1700 + 31 * channels + bs0 + 3 * bs1 + fmt, channels, bs0, bs1, S, P * K, p_short)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, fmt) for k in range(K)]
    assert any(np.isinf(to_f16(w)).any() for b in batches for w in b.wants), "no sample overflows f16"
    check_formats(ctx, batches, lambda: [L.PreviousWindowRight(case.su) for _ in range(S)], channels, fmt, SPECTRUM, memory,
                  key=key, twins=case.twins)


# ---------------------------------------------------------------------------------------------------------------------
# 3: asynchronous and prepared batches
# ---------------------------------------------------------------------------------------------------------------------
def _check_oracle(pcm, chains, wants, C, fmt, what):
    for s, (w, c) in enumerate(zip(wants, chains)):
        assert (c.status, c.n_samples) == (0, w.shape[1]), (what, s, c.status, c.n_samples)
        got = chain_pcm(pcm, c, C, fmt, w.shape[1])
        assert same_f16(got, to_f16(w)), (what, s, report(got, to_f16(w)))
    assert_guard_outside(pcm, write_mask(chains, C, fmt, pcm.size), what)


@pytest.mark.parametrize("fmt", [F16P, F16I])
def test_submits_two_deep(ctx, oracle, fmt):
    """Two host-memory batches of the same streams queued back to back (page-locked arrays), then waited on."""
    S, P, C = 6, 6, 2
    case = SpectrumCase(ctx, oracle, 1800 + fmt, C, 8, 11, S, 2 * P, 0.3)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, fmt) for k in range(2)]
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    tickets, arenas = [], []
    for b in batches:
        coeffs = ctx.host_alloc(b.coeffs.shape, np.float32)
        coeffs[...] = b.coeffs
        pcm = fill(ctx.host_alloc(b.n_out, np.float16))
        arenas.append((coeffs, pcm))
        tickets.append(ctx.submit_chains(b.chains(pwrs), SPECTRUM, HOST, coeffs, pcm, fmt))
    for k, (t, b, (_, pcm)) in enumerate(zip(tickets, batches, arenas)):
        chains = t.wait()
        _check_oracle(pcm, chains, b.wants, C, fmt, ("submit", k))
    for p, tw in zip(pwrs, case.twins):
        assert bits_equal(p.data(), tw.pwr.data())
        p.close()


def test_prepared_batch_replays_and_replans(ctx, oracle):
    """An lwb_plan in f16: planned on the first run, replayed while the streams keep their shape, re-planned after a
    reset (whose first packet emits nothing); every step against the oracle, which decodes the same packets again."""
    S, P, C = 8, 4, 2
    case = SpectrumCase(ctx, oracle, 1900, C, 8, 11, S, P, 0.0)
    b = SpectrumBatch(case, 0, P, F16P)
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    pcm = np.empty(b.n_out, np.float16)
    plan = L.Batch(ctx, b.chains(pwrs), SPECTRUM, HOST, b.coeffs, pcm, F16P)
    wants = b.wants
    for step in range(5):
        if step == 3:
            for p, tw in zip(pwrs, case.twins):
                p.reset()
                tw.pwr.reset()
        if step:
            wants = case.advance(0, P)
        fill(pcm)
        with expect_kernels(ctx, ran={"k_long"}, not_ran=ALL_KERNELS - {"k_long"}):
            plan.run()
        _check_oracle(pcm, plan.collect(), wants, C, F16P, ("step", step))
    for p, tw in zip(pwrs, case.twins):
        assert bits_equal(p.data(), tw.pwr.data())
    plan.close()
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: the front half
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,channels,floor0", [(1601, 2, False), (1602, 1, True), (1603, 6, True)])
def test_ogg_stream_reader_generic_f16(ctx, oracle, seed, channels, floor0):
    spec, packets, infos = build_stream(seed, channels, floor0, 14)
    want, _ = oracle_pcm(oracle, spec, infos)
    cut = 37
    data = vp.ogg_stream(0x1616, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets,
                         page_granules(want, 3, cut), packets_per_page=3)
    for interleaved in (False, True):
        rd = fe.OggStreamReader(ctx, data)
        for i, w in enumerate(want):
            n = w.shape[1] - (cut if i == len(want) - 1 else 0)          # end-of-stream truncation
            got = rd.read_dec_packet_generic("f16", interleaved)
            got = got.reshape(n, channels).T if interleaved else np.array(got).reshape(channels, n)
            assert got.dtype == np.float16
            assert same_f16(got, to_f16(w[:, :n])), (interleaved, i, report(got, to_f16(w[:, :n])))
        assert rd.read_dec_packet_generic("f16", interleaved) is None
        rd.close()


def test_skip_samples_linear_f16(ctx, oracle):
    n_packets, per_page, channels = 17, 3, 2
    spec, packets, infos = build_stream(1610, channels, False, n_packets)
    want, _ = oracle_pcm(oracle, spec, infos)
    gran = page_granules(want, per_page, 11)
    data = vp.ogg_stream(0x1617, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets, gran,
                         packets_per_page=per_page)
    rd = fe.OggStreamReader(ctx, data)
    model = _ReaderModel(oracle, spec, infos, gran, per_page)
    w = model.read()
    assert same_f16(np.array(rd.read_dec_packet_generic("f16")).reshape(channels, -1), to_f16(w))
    for to_skip in (3, 2500, 40, 10 ** 7):
        got, left = rd.skip_samples_linear(to_skip, sample="f16")
        w, wleft = model.skip(to_skip)
        assert left == wleft, (to_skip, left, wleft)
        if w is None:
            assert got is None
            continue
        got = np.array(got).reshape(channels, -1)
        assert got.dtype == np.float16 and same_f16(got, to_f16(w)), (to_skip, report(got, to_f16(w)))
    rd.close()


@pytest.mark.parametrize("entry", [RESIDUE, VQ])
def test_stream_batcher_f16(ctx, oracle, entry):
    channels, P, S = 2, 8, 12
    for k in range(40):                 # (a VQ batcher needs a setup lwf_headers_vq_capable accepts)
        rng = np.random.default_rng(1620 + 1000 * k)
        spec = vp.StreamSpec(rng, channels=channels)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        if entry != VQ or hdr.vq_capable():
            break
        hdr.close()
    else:
        raise AssertionError("no VQ-capable draw")
    su = hdr.make_setup(ctx)
    distinct = []
    for d in range(3):
        pkts, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, P, p_short=0.2):
            pk, info = spec.audio_packet(mode, prev, nxt)
            pkts.append(pk)
            infos.append(info)
        distinct.append((pkts, np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1)))
    stride = P * (1 << spec.bs1) // 2
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    jobs = [(pwrs[s], list(distinct[s % 3][0])) for s in range(S)]
    pcm = fill(np.empty(S * channels * stride, np.float16))
    bt = fe.StreamBatcher(ctx, hdr, threads=3, entry=entry)
    res = bt.decode(jobs, pcm, stride, out_format=F16P)
    bt.close()
    for s in range(S):
        w = distinct[s % 3][1]
        assert res[s] == (w.shape[1], P, 0), (s, res[s])
        got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, : w.shape[1]]
        assert same_f16(got, to_f16(w)), (s, report(got, to_f16(w)))
    for p in pwrs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: formats past the last one are refused, with nothing changed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [6, -1, 1 << 20])
def test_unknown_formats_are_refused_untouched(ctx, oracle, bad):
    S, P, Cn = 2, 3, 2
    case = SpectrumCase(ctx, oracle, 1630, Cn, 8, 11, S, 2 * P, 0.0, loud=False)
    b0, b1 = SpectrumBatch(case, 0, P, F16P), SpectrumBatch(case, P, 2 * P, F16P)
    pwrs = [L.PreviousWindowRight(case.su) for _ in range(S)]
    run_batch(ctx, b0, F16P, pwrs, SPECTRUM, HOST)                   # the streams hold state
    states = [p.data() for p in pwrs]
    lib = cabi.lib()
    pcm = fill(np.empty(b1.n_out, np.float16))
    arr, io = api._marshal(b1.chains(pwrs), SPECTRUM, HOST, b1.coeffs, pcm, bad, None, None, None, HOST, None)
    for i in range(S):
        arr[i].n_samples, arr[i].packets_done, arr[i].status = 1234, 56, -7

    def untouched(what):
        for i in range(S):
            assert (arr[i].n_samples, arr[i].packets_done, arr[i].status) == (1234, 56, -7), (what, i)
        for p, s in zip(pwrs, states):
            assert bits_equal(p.data(), s), what
        assert_guard_outside(pcm, np.zeros(pcm.size, bool), what)

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
        out = fill(np.empty((Cn, 2048), np.float16))
        assert lib.lwb_decode_spectrum(pwrs[0]._h, 1, 1, 1, spec.ctypes.data, bad, out.ctypes.data, 2048,
                                       ct.byref(n)) == cabi.ERR_INVALID
        assert_guard_outside(out.ravel(), np.zeros(out.size, bool), "decode_spectrum")
        untouched("decode_spectrum")
    for p in pwrs:
        p.close()
