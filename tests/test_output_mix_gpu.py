"""The output channel mix (lwb_setup_set_output_mix) on the GPU, against the oracle.

The oracle's f32 PCM is mixed by tests/mix_oracle.py (numpy float32, the library's order of operations) and converted
like any sample (i16 per samples.rs, f16 round to nearest even).  Each case also checks that:
  - the same batch without a mix gives the oracle's PCM, and a permutation or selection matrix gives exactly its bytes,
    reordered;
  - nothing outside the K-channel write set changes (sentinel-filled arenas);
  - chain results and end states (still C channels) are the unmixed run's;
  - the batch ran on k_chain, or on k_overlap for more than 8 channels and under LWB_FORCE_GENERIC=1, and both paths
    give the same bytes;
  - refused setter calls change nothing.
Covered: 2->1, 6->2, 8->8 (WAV order), 1->2 and 10->2; the spectrum, residue and VQ entries; all six formats in host
and device memory; asynchronous two-deep submits, prepared-batch replays, lwb_decode_packet / lwb_decode_spectrum; a
batch of mixed and unmixed setups; the stream batcher over a mixed header set."""
import ctypes as ct

import numpy as np
import pytest

import lewton_b200 as L
import vorbis_packer as vp
from helpers import FRONT, FUSED, GENERIC, bits_equal, environ, expect_kernels, launches_are_attributed, make_setup
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from mix_oracle import mix_f32
from test_f16_output_cpu import to_f16
from test_f16_output_gpu import (DTYPES, GUARDS, MODES, SpectrumBatch, SpectrumCase, chain_pcm, fill, planar, run_batch,
                                 same_f16)
from test_frontend_gpu import consistent_modes, oracle_pcm
from test_vq_shapes_gpu import Batch as PackerBatch
from test_vq_shapes_gpu import Streams, same_but_nan_signs

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED
F16P, F16I = cabi.OUT_F16_PLANAR, cabi.OUT_F16_INTERLEAVED
FORMATS = (F32P, I16P, F16P, F32I, I16I, F16I)
SPECTRUM, RESIDUE, VQ = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
GENERIC_ENV = {"LWB_FORCE_GENERIC": "1"}


def downmix_6_2():
    """ITU-style 5.1 -> stereo from Vorbis order FL C FR RL RR LFE (LFE dropped)."""
    a = np.float32(0.70710677)
    return np.array([[1, a, 0, a, 0, 0], [0, a, 1, 0, a, 0]], np.float32)


# name: (input channels, matrix, the input channel of each output row if the matrix is a selection / permutation)
MATRICES = {
    "2to1": (2, L.mix_mono(2), None),
    "6to2": (6, downmix_6_2(), None),
    "8to8": (8, L.mix_wav_order(8), (0, 2, 1, 7, 5, 6, 3, 4)),
    "1to2": (1, L.mix_select(1, [0, 0]), (0, 0)),
    "10to2": (10, np.random.default_rng(10).uniform(-0.6, 0.6, (2, 10)).astype(np.float32), None),
}


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


class Laid:
    """Batch b's inputs (SpectrumBatch or the VQ tests' Batch) with its chains' PCM laid out for ks[s] output channels
    of stream s: planes of n + 3 elements (planar) and gaps of 5 elements between chains, n the samples of b.wants[s] or
    sizes[s]."""

    def __init__(self, b, ks, fmt, sizes=None):
        self.b, self.ks, self.fmt = b, list(ks), fmt
        self.offs, self.strides = [], []
        o = 0
        for n, k in zip(sizes or [w.shape[1] for w in b.wants], self.ks):
            sd = n + 3 if planar(fmt) else 0
            self.offs.append(o)
            self.strides.append(sd)
            o += (k * sd if planar(fmt) else k * n) + 5
        self.n_out = o

    def __getattr__(self, name):
        return getattr(self.b, name)

    def chains(self, pwrs):
        return [L.ChainSpec(pwrs[s], m, p, n, coeff_offset=c0, packet_index=r, out_offset=o, out_stride=sd)
                for s, ((m, p, n, c0, r, _, _), o, sd) in enumerate(zip(self.b.layout, self.offs, self.strides))]

    def mask(self, chains):
        m = np.zeros(self.n_out, bool)
        for c, k in zip(chains, self.ks):
            n, o = int(c.n_samples), int(c.out_offset)
            for r in range(k if planar(self.fmt) else 1):
                s = o + r * int(c.out_stride)
                m[s:s + (n if planar(self.fmt) else n * k)] = True
        return m


def expected(oracle, w, M, fmt):
    y = w if M is None else mix_f32(w, M)
    if fmt in (F32P, F32I):
        return y
    return oracle.quantise_i16(y) if fmt in (I16P, I16I) else to_f16(y)


def same(got, want, fmt):
    if fmt in (F32P, F32I):
        return bits_equal(got, want)
    return np.array_equal(got, want) if fmt in (I16P, I16I) else same_f16(got, want)


def check_oracle(oracle, lb, pcm, chains, mats, what):
    """Every chain against the oracle's PCM of its stream, mixed by mats[s] (None: unmixed); nothing outside the write
    set changed."""
    for s, (w, c) in enumerate(zip(lb.wants, chains)):
        assert (c.status, c.n_samples) == (0, w.shape[1]), (what, s, c.status, c.n_samples, w.shape)
        got = chain_pcm(pcm, c, lb.ks[s], lb.fmt, w.shape[1])
        assert same(got, expected(oracle, w, mats[s], lb.fmt), lb.fmt), (what, s)
    u, g = GUARDS[pcm.dtype]
    bad = np.nonzero(~lb.mask(chains) & (pcm.view(u) != g))[0]
    assert not bad.size, f"{what}: {bad.size} elements outside the write set were written; first at {bad[:4]}"


def kernels_ok(delta, C, generic, what):
    if generic or C > 8:
        assert delta.get("k_overlap") and not delta.get("k_chain"), (what, delta)
    else:
        assert delta.get("k_chain") and not any(delta.get(k) for k in GENERIC | FRONT), (what, delta)
    assert not any(delta.get(k) for k in FUSED), (what, delta)


def states(pwrs):
    return [p.data() for p in pwrs]


def same_states(a, b):
    return all((x is None) == (y is None) and (x is None or bits_equal(x, y)) for x, y in zip(a, b))


def run_mixed_and_plain(ctx, oracle, batches, make_pwrs, twins, C, M, sel, entry, memory, floor_mem=HOST, what=()):
    """Every format: the batches in order on fresh streams of the unmixed setup, of the mixed setup, and of the mixed
    setup under LWB_FORCE_GENERIC=1; each checked as the module docstring says.  make_pwrs(mixed) -> streams; twins: the
    oracle streams, advanced over the batches."""
    K = M.shape[0]
    for fmt in FORMATS:
        plain, mixed, generic = make_pwrs(False), make_pwrs(True), make_pwrs(True)
        for k, b in enumerate(batches):
            w = what + (fmt, k)
            lp, lm = Laid(b, [C] * len(b.wants), fmt), Laid(b, [K] * len(b.wants), fmt)
            pcm_p, ch_p, _ = run_batch(ctx, lp, fmt, plain, entry, memory, floor_mem)
            pcm_m, ch_m, d_m = run_batch(ctx, lm, fmt, mixed, entry, memory, floor_mem)
            pcm_g, ch_g, d_g = run_batch(ctx, lm, fmt, generic, entry, memory, floor_mem, env=GENERIC_ENV)
            check_oracle(oracle, lp, pcm_p, ch_p, [None] * len(b.wants), w + ("plain",))
            check_oracle(oracle, lm, pcm_m, ch_m, [M] * len(b.wants), w + ("mixed",))
            kernels_ok(d_m, C, False, w)
            kernels_ok(d_g, C, True, w + ("generic",))
            assert same_but_nan_signs(pcm_m, pcm_g), (w, "k_chain and k_overlap differ")
            for cp, cm, cg in zip(ch_p, ch_m, ch_g):
                assert (cp.n_samples, cp.packets_done, cp.status) == (cm.n_samples, cm.packets_done, cm.status) == \
                       (cg.n_samples, cg.packets_done, cg.status), w
                if sel is not None:
                    n = int(cp.n_samples)
                    want = chain_pcm(pcm_p, cp, C, fmt, n)[list(sel)]
                    got = chain_pcm(pcm_m, cm, K, fmt, n)
                    assert np.ascontiguousarray(got).tobytes() == np.ascontiguousarray(want).tobytes(), (w, "selection")
        sp = states(plain)
        assert same_states(sp, [tw.pwr.data() for tw in twins]), (what, fmt, "end states vs oracle")
        assert same_states(sp, states(mixed)) and same_states(sp, states(generic)), (what, fmt, "end states")
        for p in plain + mixed + generic:
            p.close()


# ---------------------------------------------------------------------------------------------------------------------
# spectrum entry: every matrix, every format, host and device memory
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("name", list(MATRICES))
def test_spectrum_batches(ctx, oracle, name, memory):
    C, M, sel = MATRICES[name]
    S, P = 3, 4
    case = SpectrumCase(ctx, oracle, 2100 + C + 7 * memory, C, 8, 11, S, 2 * P, 0.3, loud=False)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, F32P) for k in range(2)]
    mixed_su = make_setup(ctx, C, 8, 11, modes=MODES)
    mixed_su.set_output_mix(M)
    assert mixed_su.output_channels == M.shape[0] and case.su.output_channels == C
    run_mixed_and_plain(ctx, oracle, batches, lambda mixed: [L.PreviousWindowRight(mixed_su if mixed else case.su) for _ in range(S)],
                        case.twins, C, M, sel, SPECTRUM, memory, what=(name, memory))


# ---------------------------------------------------------------------------------------------------------------------
# residue and VQ entries: packer bitstreams
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
@pytest.mark.parametrize("name,memory,floor_mem", [("2to1", HOST, HOST), ("6to2", DEVICE, HOST), ("8to8", HOST, DEVICE),
                                                   ("1to2", DEVICE, DEVICE)])
def test_residue_and_vq_batches(ctx, oracle, name, memory, floor_mem, entry):
    C, M, sel = MATRICES[name]
    S, P = 3, 3
    st = Streams(2200 + C, C, 8, 11, None, False, S, 2 * P, p_short=0.3)
    twins = st.twins(oracle)
    batches = [PackerBatch(st, k * P, (k + 1) * P, I16P, twins) for k in range(2)]
    plain_su = st.hdr.make_setup(ctx, floor0=st.records)
    mixed_su = st.hdr.make_setup(ctx, floor0=st.records)
    mixed_su.set_output_mix(M)
    run_mixed_and_plain(ctx, oracle, batches, lambda mixed: [L.PreviousWindowRight(mixed_su if mixed else plain_su) for _ in range(S)],
                        twins, C, M, sel, entry, memory, floor_mem, what=(name, entry, memory, floor_mem))


# ---------------------------------------------------------------------------------------------------------------------
# a batch of mixed and unmixed setups
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_mixed_and_unmixed_setups_share_a_batch(ctx, oracle, fmt):
    C, M, _ = MATRICES["6to2"]
    S, P = 6, 4
    case = SpectrumCase(ctx, oracle, 2300 + fmt, C, 8, 11, S, P, 0.3, loud=False)
    b = SpectrumBatch(case, 0, P, F32P)
    mixed_su = make_setup(ctx, C, 8, 11, modes=MODES)
    mixed_su.set_output_mix(M)
    mats = [M if s % 2 else None for s in range(S)]
    lb = Laid(b, [2 if s % 2 else C for s in range(S)], fmt)
    out = []
    for env in (None, GENERIC_ENV):
        pwrs = [L.PreviousWindowRight(mixed_su if s % 2 else case.su) for s in range(S)]
        pcm, chains, delta = run_batch(ctx, lb, fmt, pwrs, SPECTRUM, HOST, env=env)
        check_oracle(oracle, lb, pcm, chains, mats, (fmt, env))
        kernels_ok(delta, C, env is not None, (fmt, env))
        assert same_states(states(pwrs), [tw.pwr.data() for tw in case.twins]), (fmt, env, "end states")
        out.append(pcm)
        for p in pwrs:
            p.close()
    assert np.array_equal(out[0].view(np.uint8), out[1].view(np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# asynchronous submits, prepared batches, one packet
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [F32P, I16I, F16P])
def test_submits_two_deep(ctx, oracle, fmt):
    C, M, _ = MATRICES["2to1"]
    S, P = 6, 4
    case = SpectrumCase(ctx, oracle, 2400 + fmt, C, 8, 11, S, 2 * P, 0.3, loud=False)
    batches = [SpectrumBatch(case, k * P, (k + 1) * P, F32P) for k in range(2)]
    su = make_setup(ctx, C, 8, 11, modes=MODES)
    su.set_output_mix(M)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    tickets = []
    with expect_kernels(ctx, ran={"k_chain": 2}, not_ran=FUSED | GENERIC):
        for b in batches:
            lb = Laid(b, [1] * S, fmt)
            coeffs = ctx.host_alloc(b.coeffs.shape, np.float32)
            coeffs[...] = b.coeffs
            pcm = fill(ctx.host_alloc(lb.n_out, DTYPES[fmt]))
            tickets.append((lb, pcm, ctx.submit_chains(lb.chains(pwrs), SPECTRUM, HOST, coeffs, pcm, fmt)))
        for k, (lb, pcm, t) in enumerate(tickets):
            check_oracle(oracle, lb, pcm, t.wait(), [M] * S, ("submit", fmt, k))
    assert same_states(states(pwrs), [tw.pwr.data() for tw in case.twins])
    for p in pwrs:
        p.close()


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
def test_prepared_batch_replays(ctx, oracle, memory):
    """An lwb_plan of a mixed batch: planned, replayed while the streams keep their shape, re-planned after a reset."""
    C, M, _ = MATRICES["6to2"]
    S, P, fmt = 4, 4, F32P
    case = SpectrumCase(ctx, oracle, 2500 + memory, C, 8, 11, S, P, 0.0, loud=False)
    b = SpectrumBatch(case, 0, P, F32P)
    su = make_setup(ctx, C, 8, 11, modes=MODES)
    su.set_output_mix(M)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    lb = Laid(b, [2] * S, fmt, sizes=[P << 11] * S)          # room for the steady state (step 0 starts empty)
    pcm = np.empty(lb.n_out, np.float32)
    coeffs, out, frees = b.coeffs, pcm, []
    if memory == DEVICE:
        coeffs, out = ctx.device_alloc(b.coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
        ctx.h2d(coeffs, b.coeffs)
        frees = [coeffs, out]
    plan = L.Batch(ctx, lb.chains(pwrs), SPECTRUM, memory, coeffs, out, fmt)
    wants = b.wants
    for step in range(5):
        if step == 3:
            for p, tw in zip(pwrs, case.twins):
                p.reset()
                tw.pwr.reset()
        if step:
            wants = case.advance(0, P)
        fill(pcm)
        if memory == DEVICE:
            ctx.h2d(out, pcm)
        with expect_kernels(ctx, ran={"k_chain": 1}, not_ran=FUSED | GENERIC):
            plan.run()
        ctx.synchronize()
        if memory == DEVICE:
            ctx.d2h(pcm, out)
        lb.wants = wants
        check_oracle(oracle, lb, pcm, plan.collect(), [M] * S, ("plan", memory, step))
    assert same_states(states(pwrs), [tw.pwr.data() for tw in case.twins])
    plan.close()
    for p in frees:
        ctx.device_free(p)
    for p in pwrs:
        p.close()


@pytest.mark.parametrize("sample,interleaved", [("f32", False), ("i16", True), ("f16", False)])
def test_decode_packet_and_spectrum(ctx, oracle, sample, interleaved):
    """lwb_decode_packet and lwb_decode_spectrum write [K][capacity] (or [capacity][K]) of the mixed samples."""
    C, M, _ = MATRICES["6to2"]
    st = Streams(2600, C, 8, 11, None, False, 2, 6, p_short=0.3)
    twin = st.twins(oracle)[0]
    su = st.hdr.make_setup(ctx)
    su.modes = [L.ModeInfo(bf) for bf, _ in st.spec.modes]   # (read_audio_packet_generic sizes its output by them)
    su.set_output_mix(M)
    pwr = L.PreviousWindowRight(su)
    fmt = {("f32", False): F32P, ("i16", True): I16I, ("f16", False): F16P}[(sample, interleaved)]
    with expect_kernels(ctx, ran=("k_chain",), not_ran=FUSED | GENERIC):
        for pk, info, nbytes in st.packets[0]:
            w = st.oracle_packet(twin, info, nbytes)
            got = L.read_audio_packet_generic(su, st.hdr.decode_packet(pk), pwr, sample, interleaved)
            got = got.T if interleaved else got
            assert got.shape == (2, w.shape[1]) and same(got, expected(oracle, w, M, fmt), fmt), (sample, info)
    assert bits_equal(pwr.data(), twin.pwr.data())
    # the spectrum entry, on a synthetic setup
    case = SpectrumCase(ctx, oracle, 2601, C, 8, 11, 1, 5, 0.0, loud=False)
    ssu = make_setup(ctx, C, 8, 11, modes=MODES)
    ssu.set_output_mix(M)
    spwr = L.PreviousWindowRight(ssu)
    w = case.advance(0, 5)[0]
    got = np.concatenate([L.decode_spectrum(ssu, 1, case.specs[0][i], spwr, sample=sample, interleaved=interleaved)
                          for i in range(5)], axis=0 if interleaved else 1)
    got = got.T if interleaved else got
    assert got.shape == (2, w.shape[1]) and same(got, expected(oracle, w, M, fmt), fmt)
    pwr.close()
    spwr.close()


# ---------------------------------------------------------------------------------------------------------------------
# the stream batcher over a mixed header set
# ---------------------------------------------------------------------------------------------------------------------
# name: (seed, channels, blocksize_0, blocksize_1, mix or None)
BATCHER_SETS = {"six": (2701, 6, 8, 11, L.mix_wav_order(6)), "stereo": (2702, 2, 8, 11, L.mix_mono(2)),
                "mono": (2703, 1, 8, 11, None), "six_down": (2704, 6, 9, 12, downmix_6_2())}


@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
@pytest.mark.parametrize("fmt", [F32P, I16I, F16P])
def test_stream_batcher_mixed_header_set(ctx, oracle, entry, fmt):
    P = 5
    sets = []
    for name, (seed, ch, bs0, bs1, M) in BATCHER_SETS.items():
        for k in range(40):
            rng = np.random.default_rng(seed + 1000 * k)
            spec = vp.StreamSpec(rng, channels=ch, bs0=bs0, bs1=bs1, n_modes=3)
            hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
            if entry != VQ or hdr.vq_capable():
                break
            hdr.close()
        else:
            raise AssertionError("no VQ-capable draw")
        su = hdr.make_setup(ctx)
        if M is not None:
            su.set_output_mix(M)
        streams = []
        for _ in range(2):
            pk, infos = [], []
            for mode, prev, nxt in consistent_modes(spec, rng, P):
                p, info = spec.audio_packet(mode, prev, nxt, p_unused=0.15)
                pk.append(p)
                infos.append(info)
            streams.append((pk, np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1)))
        sets.append((hdr, su, M, streams))
    bt = fe.StreamBatcher(ctx, sets[0][0], threads=3, entry=entry)      # (the first set's setup needs no registering)
    for hdr, su, _, _ in sets[1:]:
        bt.add_headers(hdr, su)
    stride = P * 4096
    jobs, wants = [], []
    for hdr, su, M, streams in sets:
        for pk, w in streams:
            jobs.append((L.PreviousWindowRight(su), pk))
            wants.append((su.output_channels, M, w))
    order = np.random.default_rng(fmt).permutation(len(jobs))
    jobs, wants = [jobs[i] for i in order], [wants[i] for i in order]
    pcm = fill(np.empty(sum(k for k, _, _ in wants) * stride + 7, DTYPES[fmt]))
    res = bt.decode(jobs, pcm, stride, out_format=fmt)
    mask = np.zeros(pcm.size, bool)
    off = 0
    for j, ((k, M, w), (n, done, status)) in enumerate(zip(wants, res)):
        assert (n, done, status) == (w.shape[1], P, 0), (j, res[j])
        blk = pcm[off:off + k * stride]
        got = blk.reshape(k, stride)[:, :n] if planar(fmt) else blk[:n * k].reshape(n, k).T
        assert same(got, expected(oracle, w, M, fmt), fmt), (entry, fmt, j)
        if planar(fmt):
            for r in range(k):
                mask[off + r * stride:off + r * stride + n] = True
        else:
            mask[off:off + n * k] = True
        off += k * stride
    u, g = GUARDS[pcm.dtype]
    assert not np.any(~mask & (pcm.view(u) != g)), (entry, fmt, "written outside the jobs' samples")
    bt.close()
    for p, _ in jobs:
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# the setter's refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_setter_refusals_change_nothing(ctx, oracle):
    C, M, _ = MATRICES["6to2"]
    lib = cabi.lib()
    case = SpectrumCase(ctx, oracle, 2800, C, 8, 11, 2, 4, 0.3, loud=False)
    b = SpectrumBatch(case, 0, 4, F32P)
    su = make_setup(ctx, C, 8, 11, modes=MODES)
    su.set_output_mix(L.mix_mono(C))
    su.set_output_mix(M)                                      # a second mix replaces the first
    assert su.output_channels == 2
    bad = [(9, np.ones((9, C), np.float32)), (2, np.where(np.eye(2, C) > 0, np.float32(np.nan), np.float32(0))),
           (2, np.full((2, C), np.inf, np.float32)), (2, None), (0, np.ones((1, C), np.float32))]
    for n_out, m in bad:
        ptr = None if m is None else m.ctypes.data_as(ct.POINTER(ct.c_float))
        assert lib.lwb_setup_set_output_mix(su._h, n_out, ptr) == cabi.ERR_INVALID, n_out
        assert su.output_channels == 2
    plain = make_setup(ctx, C, 8, 11, modes=MODES)
    plain.set_output_mix(M)
    plain.set_output_mix(None)                                # cleared
    assert plain.output_channels == C
    pwrs = [L.PreviousWindowRight(su) for _ in range(2)]
    with pytest.raises(L.AudioReadError):
        su.set_output_mix(L.mix_mono(C))                      # streams are open
    with pytest.raises(L.AudioReadError):
        su.set_output_mix(None)
    assert su.output_channels == 2
    lb = Laid(b, [2, 2], F32P)
    pcm, chains, delta = run_batch(ctx, lb, F32P, pwrs, SPECTRUM, HOST)
    check_oracle(oracle, lb, pcm, chains, [M, M], "after refusals")
    kernels_ok(delta, C, False, "after refusals")
    for p in pwrs:
        p.close()
