"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs.  Bar (north_star): f32 PCM bit-identical (modulo sign of zero / NaN payload), i16 PCM
bit-identical."""
import os

import numpy as np
import pytest

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import (ALL_KERNELS, FRONT, GENERIC, RefStream, assert_contained, bits_equal, expect_kernels, fill_guard,
                     launches_are_attributed, make_setup, mismatch_report, mode_sequence, random_floor1, random_floor1_y,
                     write_set)

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------
# inverse MDCT alone (imdct.rs:291), through the post-MDCT debug tap
# ------------------------------------------------------------------------------------------------
def imdct_via_tap(ctx, bs, spectra):
    su = make_setup(ctx, 1, bs, bs, modes=((1, 0),))
    pwr = L.PreviousWindowRight(su)
    out = []
    for sp in spectra:
        pk = L.DecodedPacket(0, sp[None, :], [np.ones(len(sp), np.float32)])
        _, pre, post = L.debug_taps(su, pk, pwr)
        assert bits_equal(pre[0], sp)          # 1.0 * x is exact
        out.append(post[0])
    return out


@pytest.mark.parametrize("bs", range(6, 14))
def test_imdct_all_blocksizes_bit_exact(ctx, oracle, bs):
    rng = np.random.default_rng(1000 + bs)
    n2 = (1 << bs) // 2
    spectra = [rng.standard_normal(n2).astype(np.float32) * s for s in (1.0, 1e-2, 1e3)]
    spectra.append(np.zeros(n2, np.float32))
    e = np.zeros(n2, np.float32)
    e[n2 // 3] = 1.0
    spectra.append(e)
    for sp, got in zip(spectra, imdct_via_tap(ctx, bs, spectra)):
        want = oracle.inverse_mdct(sp, bs)
        assert bits_equal(got, want), mismatch_report(got, want)


def test_imdct_reference_kat(ctx):
    """The reference's own KATs (imdct_test.rs) through the GPU path, at the reference's tolerance."""
    import json
    with open(os.path.join(os.path.dirname(__file__), "golden", "imdct_kat.json")) as f:
        kat = {k: np.array([np.float32(v) for v in a], np.float32) for k, a in json.load(f)["arrays"].items()}
    for idx, bs, eps in ((1, 8, 5e-5), (2, 8, 5e-5), (3, 11, 5e-4)):
        got = imdct_via_tap(ctx, bs, [kat[f"IMDCT_INPUT_TEST_ARR_{idx}"]])[0]
        want = kat[f"IMDCT_OUTPUT_TEST_ARR_{idx}"]
        assert int(np.sum(np.abs(got - want) >= np.float32(eps))) == 0


# ------------------------------------------------------------------------------------------------
# packet by packet, spectrum entry: window geometry, OLA, state, formats (audio.rs:1041-1157)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channels,bs0,bs1,seed", [(1, 8, 11, 0), (2, 8, 11, 1), (6, 8, 11, 2), (2, 6, 9, 3),
                                                   (1, 7, 13, 4), (3, 10, 10, 5)])
def test_packet_sequence_mixed_blocks(ctx, oracle, channels, bs0, bs1, seed):
    rng = np.random.default_rng(seed)
    su = make_setup(ctx, channels, bs0, bs1)
    pwr = L.PreviousWindowRight(su)
    ref = RefStream(oracle, channels, bs0, bs1, [(0, 0), (1, 0)])
    modes, prev, nxt = mode_sequence(rng, 14)
    assert pwr.is_empty()
    for i in range(len(modes)):
        n2 = (1 << (bs1 if modes[i] else bs0)) // 2
        spec = (rng.standard_normal((channels, n2)) * 0.1).astype(np.float32)
        rc, want = ref.spectrum(int(modes[i]), int(prev[i]), int(nxt[i]), spec)
        assert L.get_decoded_sample_count(su, int(modes[i]), prev[i], nxt[i]) == \
            (want.shape[1] if i else L.get_decoded_sample_count(su, int(modes[i]), prev[i], nxt[i]))
        if rc:
            with pytest.raises(L.AudioReadError) as e:
                L.decode_spectrum(su, int(modes[i]), spec, pwr, prev[i], nxt[i])
            assert e.value.kind == "AudioBadFormat"
            assert pwr.is_empty() and ref.pwr.is_empty()
            continue
        fmt = i % 4
        if fmt == 0:
            got = L.decode_spectrum(su, int(modes[i]), spec, pwr, prev[i], nxt[i])
            assert bits_equal(got, want), mismatch_report(got, want)
        elif fmt == 1:
            got = L.decode_spectrum(su, int(modes[i]), spec, pwr, prev[i], nxt[i], sample="i16")
            assert np.array_equal(got, oracle.quantise_i16(want))
        elif fmt == 2:
            got = L.decode_spectrum(su, int(modes[i]), spec, pwr, prev[i], nxt[i], interleaved=True)
            assert bits_equal(got, want.T)
        else:
            got = L.decode_spectrum(su, int(modes[i]), spec, pwr, prev[i], nxt[i], sample="i16", interleaved=True)
            assert np.array_equal(got, oracle.quantise_i16(want).T)
        assert len(pwr) == len(ref.pwr)
        assert bits_equal(pwr.data(), ref.pwr.data())


def test_first_packet_and_reset_semantics(ctx, oracle):
    """audio.rs:1140-1151: no previous half -> 0 samples; reset/clone behave like the Rust type."""
    rng = np.random.default_rng(7)
    su = make_setup(ctx, 2, 8, 11)
    pwr = L.PreviousWindowRight.new(su)
    spec = rng.standard_normal((2, 1024)).astype(np.float32)
    out = L.decode_spectrum(su, 1, spec, pwr)
    assert out.shape == (2, 0) and not pwr.is_empty() and len(pwr) == 1024
    x = np.stack([oracle.inverse_mdct(spec[c], 11) for c in range(2)])
    assert bits_equal(pwr.data(), x[:, 1024:])
    twin = pwr.clone()
    a = L.decode_spectrum(su, 1, spec, pwr)
    b = L.decode_spectrum(su, 1, spec, twin)
    assert a.shape == (2, 1024) and bits_equal(a, b)
    pwr.reset()
    assert pwr.is_empty()
    assert L.decode_spectrum(su, 1, spec, pwr).shape == (2, 0)


def test_ola_guard_is_bad_format_and_empties_state(ctx, oracle):
    """audio.rs:1107-1111 (fuzzing regression): slope shorter than the previous half."""
    rng = np.random.default_rng(8)
    su = make_setup(ctx, 1, 8, 11)
    pwr = L.PreviousWindowRight(su)
    L.decode_spectrum(su, 1, rng.standard_normal((1, 1024)).astype(np.float32), pwr)      # long, next=long
    with pytest.raises(L.AudioReadError) as e:
        L.decode_spectrum(su, 0, rng.standard_normal((1, 128)).astype(np.float32), pwr)    # short follows
    assert e.value.kind == "AudioBadFormat" and pwr.is_empty()
    with pytest.raises(L.AudioReadError) as e:
        L.decode_spectrum(su, 7, np.zeros((1, 128), np.float32), pwr)                      # audio.rs:926-930
    assert e.value.kind == "AudioBadFormat"


# ------------------------------------------------------------------------------------------------
# full packets: coupling + floor-1 + multiply (audio.rs:988-1039)
# ------------------------------------------------------------------------------------------------
def _random_packet_case(rng, channels, bs0, bs1):
    n2s = ((1 << bs0) // 2, (1 << bs1) // 2)
    floors = [random_floor1(rng, n2s[1]) for _ in range(3)]
    steps = []
    for _ in range(int(rng.integers(0, 2 * channels))):
        m, a = rng.choice(channels, 2, replace=False) if channels > 1 else (0, 0)
        if m != a:
            steps.append((int(m), int(a)))
    mappings = [{"coupling": steps, "floor_of_channel": [int(rng.integers(0, 3)) for _ in range(channels)]},
                {"coupling": [], "floor_of_channel": [0] * channels}]
    modes = [(0, 0), (1, 0), (1, 1), (0, 1)]
    return floors, mappings, modes


@pytest.mark.parametrize("channels,bs0,bs1,seed", [(2, 8, 11, 10), (6, 8, 11, 11), (1, 6, 8, 12), (12, 7, 10, 13),
                                                   (3, 9, 13, 14)])
def test_full_packets_coupling_and_floor1(ctx, oracle, channels, bs0, bs1, seed):
    rng = np.random.default_rng(seed)
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwr = L.PreviousWindowRight(su)
    ref = RefStream(oracle, channels, bs0, bs1, modes, mappings, floors)
    bf, prev, nxt = mode_sequence(rng, 10)
    for i in range(len(bf)):
        mode = int(rng.choice([m for m in range(4) if modes[m][0] == bf[i]]))
        n2 = (1 << (bs1 if bf[i] else bs0)) // 2
        # sparse, signed residue with exact zeros (exercises all inverse_couple branches)
        res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
        mp = mappings[modes[mode][1]]
        fl = []
        for c in range(channels):
            r = rng.random()
            if r < 0.2:
                fl.append(None)
            elif r < 0.3:
                fl.append(rng.random(n2).astype(np.float32))
            else:
                mult, xs = floors[mp["floor_of_channel"][c]]
                fl.append(random_floor1_y(rng, mult, len(xs), wild=(seed % 2 == 0)))
        rc, want = ref.packet(mode, int(prev[i]), int(nxt[i]), res, fl)
        pk = L.DecodedPacket(mode, res, fl, prev[i], nxt[i])
        if rc:
            with pytest.raises(L.AudioReadError):
                L.read_audio_packet_generic(su, pk, pwr)
            assert pwr.is_empty() == ref.pwr.is_empty()
            continue
        if i % 2:
            got = L.read_audio_packet(su, pk, pwr)                  # Vec<Vec<i16>>
            assert np.array_equal(got, oracle.quantise_i16(want))
        else:
            got = L.read_audio_packet_generic(su, pk, pwr)
            assert bits_equal(got, want), mismatch_report(got, want)
        assert bits_equal(pwr.data(), ref.pwr.data())


def test_debug_taps_match_oracle_stages(ctx, oracle):
    """record_residue_post_inverse / record_pre_mdct / record_post_mdct (audio.rs:1004,1041,1054)."""
    rng = np.random.default_rng(21)
    channels, bs0, bs1 = 4, 8, 11
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    mappings[0]["coupling"] = [(0, 1), (2, 3), (0, 2)]          # chain through a shared channel
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwr = L.PreviousWindowRight(su)
    res = (rng.standard_normal((channels, 1024)) * rng.integers(0, 2, (channels, 1024))).astype(np.float32)
    fl = [random_floor1_y(rng, *(lambda f: (f[0], len(f[1])))(floors[mappings[0]["floor_of_channel"][c]]))
          for c in range(channels)]
    post_inv, pre, post = L.debug_taps(su, L.DecodedPacket(1, res, fl), pwr)
    r = res.copy()
    for m, a in reversed(mappings[0]["coupling"]):
        r[m], r[a] = oracle.inverse_couple(r[m], r[a])
    assert bits_equal(post_inv, r)
    for c in range(channels):
        mult, xs = floors[mappings[0]["floor_of_channel"][c]]
        ofl = oracle.make_floor1(mult, xs)
        fy, s2 = oracle.floor1_amplitude(ofl, fl[c])
        curve = oracle.floor1_synthesis(ofl, fy, s2, 1024)
        assert bits_equal(pre[c], curve * r[c]), c
        assert bits_equal(post[c], oracle.inverse_mdct(pre[c], 11))
    assert pwr.is_empty()                                         # taps do not touch the state


# ------------------------------------------------------------------------------------------------
# batches (lwb_decode_chains): generic and fused paths, host and device memory
# ------------------------------------------------------------------------------------------------
def run_batch(ctx, su, pwrs, spec, n_packets, memory, env=None):
    """spec [S][P][C][1024] -> pcm [S][C][P*1024] (planar f32), all long/long."""
    S, P, C, n2 = spec.shape
    stride = P * n2
    chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * C * n2, out_offset=s * C * stride,
                          out_stride=stride) for s in range(S)]
    pcm = np.zeros((S, C, stride), np.float32)
    old = {}
    for k, v in (env or {}).items():
        old[k] = os.environ.get(k)
        os.environ[k] = v
    try:
        if memory == cabi.MEM_HOST:
            L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, spec, pcm, cabi.OUT_F32_PLANAR)
        else:
            d_in = ctx.device_alloc(spec.nbytes)
            d_out = ctx.device_alloc(pcm.nbytes)
            ctx.h2d(d_out, pcm)
            ctx.h2d(d_in, spec)
            L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, d_in, d_out, cabi.OUT_F32_PLANAR)
            ctx.synchronize()
            ctx.d2h(pcm, d_out)
            ctx.device_free(d_in)
            ctx.device_free(d_out)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    return chains, pcm


def long_batch_kernels(env):
    """expect_kernels arguments for a uniform long spectrum batch run under `env` (see run_batch)."""
    fg = (env or {}).get("LWB_FORCE_GENERIC")
    ran = {"k_imdct", "k_overlap", "k_save_state"} if fg == "1" else {"k_chain"} if fg else {"k_long"}
    return dict(ran=ran, not_ran=ALL_KERNELS - ran)


def oracle_batch(oracle, spec, states=None):
    S, P, C, n2 = spec.shape
    outs, finals = [], []
    for s in range(S):
        pwr = oracle.Pwr(C, 11)
        if states is not None and states[s] is not None:
            pwr.set_data(states[s])
        parts = []
        for p in range(P):
            rc, pcm = oracle.synth_spectrum(8, 11, 1, 1, 1, spec[s, p], pwr)
            assert rc == 0
            parts.append(pcm)
        outs.append(np.concatenate(parts, axis=1))
        finals.append(pwr.data())
    return outs, finals


@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
@pytest.mark.parametrize("env", [None, {"LWB_FORCE_GENERIC": "1"}, {"LWB_FORCE_GENERIC": "2"},
                                 {"LWB_LONG_TARGET_RUNS": "100000"}])
def test_batch_long_blocks_vs_oracle(ctx, oracle, memory, env):
    """S stereo streams x P long blocks, fresh streams then a second batch that continues them;
    fused path, fused path with forced run cuts (primer packets), and the generic path."""
    rng = np.random.default_rng(31)
    S, P, C = 5, 19, 2
    su = make_setup(ctx, C, 8, 11)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    spec1 = (rng.standard_normal((S, P, C, 1024)) * 0.05).astype(np.float32)
    spec2 = (rng.standard_normal((S, P, C, 1024)) * 0.05).astype(np.float32)
    with expect_kernels(ctx, **long_batch_kernels(env)):
        chains, pcm1 = run_batch(ctx, su, pwrs, spec1, P, memory, env)
    want1, st1 = oracle_batch(oracle, spec1)
    for s in range(S):
        assert chains[s].status == 0 and chains[s].packets_done == P and chains[s].n_samples == (P - 1) * 1024
        assert bits_equal(pcm1[s][:, : (P - 1) * 1024], want1[s]), (s, mismatch_report(pcm1[s][:, : (P - 1) * 1024], want1[s]))
        assert bits_equal(pwrs[s].data(), st1[s])
    with expect_kernels(ctx, **long_batch_kernels(env)):
        chains, pcm2 = run_batch(ctx, su, pwrs, spec2, P, memory, env)
    want2, st2 = oracle_batch(oracle, spec2, st1)
    for s in range(S):
        assert chains[s].n_samples == P * 1024
        assert bits_equal(pcm2[s], want2[s]), (s, mismatch_report(pcm2[s], want2[s]))
        assert bits_equal(pwrs[s].data(), st2[s])


def test_fused_path_with_imported_asymmetric_state(ctx, oracle):
    """A state that did not come from a long block (not mirror-symmetric) must still be honoured."""
    rng = np.random.default_rng(33)
    su = make_setup(ctx, 1, 8, 11)
    pwr = L.PreviousWindowRight(su)
    st = rng.standard_normal((1, 1024)).astype(np.float32)
    pwr.set_data(st)
    spec = rng.standard_normal((1, 3, 1, 1024)).astype(np.float32)
    _, pcm = run_batch(ctx, su, [pwr], spec, 3, cabi.MEM_HOST)
    want, fin = oracle_batch(oracle, spec, [st])
    assert bits_equal(pcm[0], want[0]) and bits_equal(pwr.data(), fin[0])


def test_fused_and_generic_agree_at_scale(ctx, oracle):
    """Size-independent property at a larger size: the fused kernel and the generic path are
    two independent schedules of the same arithmetic and must agree bit for bit; a sample of
    chains is also checked against the oracle."""
    rng = np.random.default_rng(35)
    S, P, C = 96, 24, 2
    su = make_setup(ctx, C, 8, 11)
    spec = (rng.standard_normal((S, P, C, 1024)) * 0.02).astype(np.float32)
    pa = [L.PreviousWindowRight(su) for _ in range(S)]
    pb = [L.PreviousWindowRight(su) for _ in range(S)]
    with expect_kernels(ctx, **long_batch_kernels(None)):
        _, fused = run_batch(ctx, su, pa, spec, P, cabi.MEM_DEVICE)
    with expect_kernels(ctx, **long_batch_kernels({"LWB_FORCE_GENERIC": "1"})):
        _, generic = run_batch(ctx, su, pb, spec, P, cabi.MEM_DEVICE, {"LWB_FORCE_GENERIC": "1"})
    assert np.array_equal(fused.view(np.uint32), generic.view(np.uint32))
    want, _ = oracle_batch(oracle, spec[:3])
    for s in range(3):
        assert bits_equal(fused[s][:, : (P - 1) * 1024], want[s])
    # linearity of the whole path in exact arithmetic: scaling the input by 2 scales the output by 2
    pc = [L.PreviousWindowRight(su) for _ in range(S)]
    with expect_kernels(ctx, **long_batch_kernels(None)):
        _, doubled = run_batch(ctx, su, pc, spec * np.float32(2), P, cabi.MEM_DEVICE)
    assert np.array_equal(doubled.view(np.uint32), (fused * np.float32(2)).view(np.uint32))


def test_batch_mixed_blocks_residue_entry(ctx, oracle):
    """Chains with mixed short/long packets, coupling and floor-1, i16 interleaved output."""
    rng = np.random.default_rng(37)
    channels, bs0, bs1, S, P = 2, 8, 11, 4, 9
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    mappings[0]["coupling"] = [(0, 1)]
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [RefStream(oracle, channels, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    coeffs, kinds, ys, specs, want = [], [], [], [], []
    chains = []
    coeff_off = pkt_idx = out_off = 0
    for s in range(S):
        bf, prev, nxt = mode_sequence(rng, P, p_short=0.4)
        mode_ids = np.array([0 if not b else 1 for b in bf], np.uint8)
        total = 0
        parts = []
        c_off0, p_idx0 = coeff_off, pkt_idx
        for i in range(P):
            n2 = (1 << (bs1 if bf[i] else bs0)) // 2
            res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
            fl = []
            for c in range(channels):
                mult, xs = floors[mappings[0]["floor_of_channel"][c]]
                fl.append(None if rng.random() < 0.15 else random_floor1_y(rng, mult, len(xs)))
            rc, pcm = refs[s].packet(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res, fl)
            assert rc == 0
            parts.append(pcm)
            total += pcm.shape[1]
            coeffs.append(res.ravel())
            k, y, _ = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
            kinds.append(k)
            ys.append(y)
            coeff_off += res.size
            pkt_idx += 1
        want.append(np.concatenate(parts, axis=1))
        chains.append(L.ChainSpec(pwrs[s], mode_ids, prev, nxt, coeff_offset=c_off0, packet_index=p_idx0,
                                  out_offset=out_off, out_stride=0))
        out_off += total * channels
    coeffs = np.concatenate(coeffs)
    kinds = np.concatenate(kinds)
    ys = np.concatenate(ys)
    pcm = np.zeros(out_off, np.int16)
    L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, coeffs, pcm, cabi.OUT_I16_INTERLEAVED,
                    floor_kind=kinds, floor1_y=ys)
    pos = 0
    for s in range(S):
        n = want[s].shape[1]
        assert chains[s].status == 0 and chains[s].n_samples == n
        got = pcm[pos: pos + n * channels].reshape(n, channels)
        assert np.array_equal(got, oracle.quantise_i16(want[s]).T), s
        pos += n * channels
        assert bits_equal(pwrs[s].data(), refs[s].pwr.data())


def test_batch_error_mid_chain(ctx, oracle):
    """A chain whose 3rd packet trips the OLA guard: earlier packets are decoded, the chain
    reports AudioBadFormat at index 2 and the stream ends up empty (audio.rs:1083,1107-1111)."""
    rng = np.random.default_rng(39)
    su = make_setup(ctx, 1, 8, 11)
    pwr = L.PreviousWindowRight(su)
    modes = np.array([1, 1, 0, 1], np.uint8)           # long, long(next=long), short -> guard
    spec = rng.standard_normal(1024 * 2 + 128 + 1024).astype(np.float32)
    pcm = np.zeros(4096, np.float32)
    ch = L.ChainSpec(pwr, modes, out_stride=4096)
    L.decode_chains(ctx, [ch], cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, spec, pcm, cabi.OUT_F32_PLANAR)
    assert ch.status == cabi.ERR_BAD_FORMAT and ch.packets_done == 2 and ch.n_samples == 1024
    assert pwr.is_empty()
    ref = oracle.Pwr(1, 11)
    oracle.synth_spectrum(8, 11, 1, 1, 1, spec[None, :1024], ref)
    _, want = oracle.synth_spectrum(8, 11, 1, 1, 1, spec[None, 1024:2048], ref)
    assert bits_equal(pcm[:1024], want[0])


def test_special_values_on_gpu(ctx, oracle):
    """Denormals are kept (no flush-to-zero), inf/NaN propagate like on the CPU."""
    rng = np.random.default_rng(41)
    su = make_setup(ctx, 1, 8, 11)
    spec = rng.standard_normal((2, 4, 1, 1024)).astype(np.float32)
    spec[0, 0, 0, :100] = 1e-42          # denormal inputs
    spec[0, 1, 0] *= 1e-38               # outputs around / below the normal range
    spec[0, 2, 0] *= 1e-41
    spec[0, 3, 0] = 0.0
    spec[1, 1, 0, 3] = np.inf            # second stream: inf / NaN
    spec[1, 2, 0, 9] = np.nan
    want, fin = oracle_batch(oracle, spec)
    assert np.any((np.abs(want[0]) > 0) & (np.abs(want[0]) < 1.1e-38)), "test should exercise denormal outputs"
    assert np.any(np.isnan(want[1]))
    for env in (None, {"LWB_FORCE_GENERIC": "1"}, {"LWB_FORCE_GENERIC": "2"}):
        pwrs = [L.PreviousWindowRight(su) for _ in range(2)]
        with expect_kernels(ctx, **long_batch_kernels(env)):
            _, pcm = run_batch(ctx, su, pwrs, spec, 4, cabi.MEM_HOST, env)
        for s in range(2):
            assert bits_equal(pcm[s][:, :3072], want[s]), (env, s, mismatch_report(pcm[s][:, :3072], want[s]))
            assert bits_equal(pwrs[s].data(), fin[s])


@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
def test_fused_i16_planar_output(ctx, oracle, memory):
    """Vec<Vec<i16>> (samples.rs:92-103) straight out of the fused kernel: bit-exact after the quantise."""
    rng = np.random.default_rng(51)
    S, P, C = 6, 11, 2
    su = make_setup(ctx, C, 8, 11)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    spec = (rng.standard_normal((S, P, C, 1024)) * 0.4).astype(np.float32)     # loud: exercises the clamp
    spec[4, 2, 0] *= 1e6                 # far out of range on both sides
    spec[5, 3, 0, 7] = np.inf            # +-inf and NaN samples (NaN -> 0, samples.rs:92-103 `as i16`)
    spec[5, 6, 1, 9] = np.nan
    stride = P * 1024
    chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * C * 1024, out_offset=s * C * stride,
                          out_stride=stride) for s in range(S)]
    pcm = np.zeros((S, C, stride), np.int16)
    if memory == cabi.MEM_HOST:
        with expect_kernels(ctx, **long_batch_kernels(None)):
            L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, spec, pcm, cabi.OUT_I16_PLANAR)
    else:
        d_in, d_out = ctx.device_alloc(spec.nbytes), ctx.device_alloc(pcm.nbytes)
        ctx.h2d(d_in, spec)
        ctx.h2d(d_out, pcm)
        with expect_kernels(ctx, **long_batch_kernels(None)):
            L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, d_in, d_out, cabi.OUT_I16_PLANAR)
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        ctx.device_free(d_in)
        ctx.device_free(d_out)
    want, fin = oracle_batch(oracle, spec)
    assert any(np.any(np.abs(w) > 1.0) for w in want), "test should exercise the i16 clamp"
    assert np.any(np.isnan(want[5])) and np.any(np.abs(want[4]) > 1e3)
    for s in range(S):
        assert chains[s].n_samples == (P - 1) * 1024
        assert np.array_equal(pcm[s][:, : (P - 1) * 1024], oracle.quantise_i16(want[s])), s
        assert bits_equal(pwrs[s].data(), fin[s])


@pytest.mark.parametrize("memory,fmt", [(cabi.MEM_HOST, "f32"), (cabi.MEM_DEVICE, "f32"), (cabi.MEM_HOST, "i16")])
def test_residue_entry_long_batch_uses_prologue_plus_fused(ctx, oracle, memory, fmt):
    """Full packets (coupling + floor-1 + multiply) in uniform long batches: k_prologue forms the
    spectrum, the fused kernel does IMDCT/window/OLA.  Two consecutive batches (second one overlaps
    with the stream state)."""
    rng = np.random.default_rng(53)
    channels, bs0, bs1, S, P = 2, 8, 11, 5, 9
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    mappings[0]["coupling"] = [(0, 1)]
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [RefStream(oracle, channels, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    with expect_kernels(ctx, ran={"k_floor1_segments": 2, "k_prologue_fused": 2, "k_long": 2},
                        not_ran=ALL_KERNELS - FRONT - {"k_long"}):
        for batch in range(2):
            res = (rng.standard_normal((S, P, channels, 1024)) * rng.integers(0, 2, (S, P, channels, 1024))).astype(np.float32)
            kinds = np.zeros((S, P, channels), np.uint8)
            ys = np.zeros((S, P, channels, cabi.MAX_POSTS), np.uint32)
            want = []
            for s in range(S):
                parts = []
                for p in range(P):
                    fl = []
                    for c in range(channels):
                        mult, xs = floors[mappings[0]["floor_of_channel"][c]]
                        fl.append(None if rng.random() < 0.1 else random_floor1_y(rng, mult, len(xs)))
                    k, y, _ = L.DecodedPacket(1, res[s, p], fl).pack()
                    kinds[s, p], ys[s, p] = k, y
                    rc, pcm = refs[s].packet(1, 1, 1, res[s, p], fl)
                    assert rc == 0
                    parts.append(pcm)
                want.append(np.concatenate(parts, axis=1))
            stride = P * 1024
            chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * channels * 1024, packet_index=s * P,
                                  out_offset=s * channels * stride, out_stride=stride) for s in range(S)]
            dt = np.float32 if fmt == "f32" else np.int16
            of = cabi.OUT_F32_PLANAR if fmt == "f32" else cabi.OUT_I16_PLANAR
            pcm = np.zeros((S, channels, stride), dt)
            if memory == cabi.MEM_HOST:
                L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, res, pcm, of, floor_kind=kinds, floor1_y=ys)
            else:
                d_in, d_out = ctx.device_alloc(res.nbytes), ctx.device_alloc(pcm.nbytes)
                ctx.h2d(d_in, res)
                ctx.h2d(d_out, pcm)
                L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, d_in, d_out, of, floor_kind=kinds, floor1_y=ys)
                ctx.synchronize()
                ctx.d2h(pcm, d_out)
                ctx.device_free(d_in)
                ctx.device_free(d_out)
            for s in range(S):
                n = want[s].shape[1]
                assert chains[s].status == 0 and chains[s].n_samples == n
                if fmt == "f32":
                    assert bits_equal(pcm[s][:, :n], want[s]), (batch, s, mismatch_report(pcm[s][:, :n], want[s]))
                else:
                    assert np.array_equal(pcm[s][:, :n], oracle.quantise_i16(want[s])), (batch, s)
                assert bits_equal(pwrs[s].data(), refs[s].pwr.data())
        # 2 batches x (k_floor1_segments + k_prologue_fused + fused kernel): the generic IMDCT/overlap kernels did not run


def test_prepared_batch_reuses_descriptors_and_replans_on_state_change(ctx, oracle):
    """lwb_plan_*: same results as lwb_decode_chains across state transitions (empty -> history),
    a reset of one stream in between (forces a re-plan), and many steady-state executions."""
    rng = np.random.default_rng(57)
    S, P, C = 6, 9, 2
    su = make_setup(ctx, C, 8, 11)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [oracle.Pwr(C, 11) for _ in range(S)]
    spec = np.zeros((S, P, C, 1024), np.float32)
    stride = P * 1024
    pcm = np.zeros((S, C, stride), np.float32)
    d_in, d_out = ctx.device_alloc(spec.nbytes), ctx.device_alloc(pcm.nbytes)
    chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * C * 1024, out_offset=s * C * stride,
                          out_stride=stride) for s in range(S)]
    batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, d_in, d_out, cabi.OUT_F32_PLANAR)
    for it in range(6):
        spec[:] = (rng.standard_normal(spec.shape) * 0.05).astype(np.float32)
        if it == 3:
            pwrs[2].reset()
            refs[2].reset()
        ctx.h2d(d_in, spec)
        ctx.h2d(d_out, np.zeros_like(pcm))
        batch.run()
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        batch.collect()
        for s in range(S):
            parts = []
            for p in range(P):
                rc, o = oracle.synth_spectrum(8, 11, 1, 1, 1, spec[s, p], refs[s])
                assert rc == 0
                parts.append(o)
            want = np.concatenate(parts, axis=1)
            assert chains[s].n_samples == want.shape[1] and chains[s].status == 0, (it, s)
            assert bits_equal(pcm[s][:, : want.shape[1]], want), (it, s)
            assert bits_equal(pwrs[s].data(), refs[s].data())
    batch.close()
    ctx.device_free(d_in)
    ctx.device_free(d_out)


def test_full_bench_size_exact_by_replication(ctx, oracle):
    """BASELINE full size (4096 stereo streams x 16 long packets per step, 1 GiB of I/O): the batch
    is 512 copies of 8 distinct base streams, so every one of the 4096 outputs must be bit-identical
    to the oracle's output for its base stream -- an exact check at full size at 1/512 of the oracle
    cost ("checksum of checksums").  Two steps: fresh streams, then with history."""
    rng = np.random.default_rng(61)
    S, P, C, B = 4096, 16, 2, 8
    su = make_setup(ctx, C, 8, 11)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    stride = P * 1024
    d_in, d_out = ctx.device_alloc(S * P * C * 1024 * 4), ctx.device_alloc(S * C * stride * 4)
    chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * C * 1024, out_offset=s * C * stride,
                          out_stride=stride) for s in range(S)]
    batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, d_in, d_out, cabi.OUT_F32_PLANAR)
    refs = [oracle.Pwr(C, 11) for _ in range(B)]
    pcm = np.zeros((S, C, stride), np.float32)
    for step in range(2):
        base = (rng.standard_normal((B, P, C, 1024)) * 1e-2).astype(np.float32)
        spec = np.ascontiguousarray(np.tile(base, (S // B, 1, 1, 1)))          # stream s uses base s % B
        ctx.h2d(d_in, spec)
        ctx.h2d(d_out, np.zeros_like(pcm))
        batch.run()
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        want = []
        for b in range(B):
            parts = [oracle.synth_spectrum(8, 11, 1, 1, 1, base[b, p], refs[b])[1] for p in range(P)]
            want.append(np.concatenate(parts, axis=1))
        n = want[0].shape[1]
        assert n == (P - 1 + step) * 1024
        got = pcm[:, :, :n].reshape(S // B, B, C, n)
        for b in range(B):
            assert np.array_equal(got[:, b].view(np.uint32), np.broadcast_to(want[b].view(np.uint32), (S // B, C, n))), (step, b)
    for s in (0, 1, 7, 4095):
        assert bits_equal(pwrs[s].data(), refs[s % B].data())
    batch.close()
    ctx.device_free(d_in)
    ctx.device_free(d_out)


@pytest.mark.parametrize("channels,bs0,bs1,fmt,seed", [(2, 8, 11, cabi.OUT_F32_PLANAR, 70), (6, 8, 11, cabi.OUT_I16_INTERLEAVED, 71),
                                                       (1, 6, 13, cabi.OUT_F32_INTERLEAVED, 72), (8, 7, 9, cabi.OUT_I16_PLANAR, 73)])
def test_chain_kernel_vs_four_kernel_path_mixed_sequences(ctx, oracle, channels, bs0, bs1, fmt, seed):
    """The chain kernel (one launch, shared-memory resident) and the four-kernel path are independent
    schedules of the same arithmetic: bit-identical on random mixed short/long chains with full
    packets (coupling + floor-1 / dense / unused floors), and both equal to the oracle."""
    rng = np.random.default_rng(seed)
    S, P = 5, 12
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    refs = [RefStream(oracle, channels, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    coeffs, dense, kinds, ys, want, seqs = [], [], [], [], [], []
    for s in range(S):
        bf, prev, nxt = mode_sequence(rng, P, p_short=0.45)
        mode_ids = np.array([int(rng.choice([m for m in range(4) if modes[m][0] == b])) for b in bf], np.uint8)
        parts = []
        for i in range(P):
            n2 = (1 << (bs1 if bf[i] else bs0)) // 2
            res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
            mp = mappings[modes[mode_ids[i]][1]]
            fl = []
            for c in range(channels):
                mult, xs = floors[mp["floor_of_channel"][c]]
                r = rng.random()
                fl.append(None if r < 0.15 else (rng.random(n2).astype(np.float32) if r < 0.25
                                                 else random_floor1_y(rng, mult, len(xs))))
            rc, pcm = refs[s].packet(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res, fl)
            assert rc == 0
            parts.append(pcm)
            k, y, d = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
            coeffs.append(res.ravel())
            dense.append((d if d is not None else np.zeros_like(res)).ravel())
            kinds.append(k)
            ys.append(y)
        want.append(np.concatenate(parts, axis=1))
        seqs.append((mode_ids, prev, nxt))
    coeffs, dense = np.concatenate(coeffs), np.concatenate(dense)
    kinds, ys = np.concatenate(kinds), np.concatenate(ys)
    outs = {}
    interleaved = fmt in (cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED)
    dt = np.float32 if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED) else np.int16
    for name, env in (("chain", None), ("four", {"LWB_FORCE_GENERIC": "1"})):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        chains, coeff_off, out_off = [], 0, 0
        for s in range(S):
            n = want[s].shape[1]
            mode_ids, prev, nxt = seqs[s]
            chains.append(L.ChainSpec(pwrs[s], mode_ids, prev, nxt, coeff_offset=coeff_off, packet_index=s * P,
                                      out_offset=out_off, out_stride=0 if interleaved else n))
            coeff_off += sum(channels * ((1 << (bs1 if modes[m][0] else bs0)) // 2) for m in mode_ids)
            out_off += n * channels
        pcm = np.zeros(out_off, dt)
        old = os.environ.get("LWB_FORCE_GENERIC")
        if env:
            os.environ.update(env)
        try:
            L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, coeffs, pcm, fmt, floor_kind=kinds, floor1_y=ys,
                            dense_floor=dense)
        finally:
            if env:
                if old is None:
                    del os.environ["LWB_FORCE_GENERIC"]
                else:
                    os.environ["LWB_FORCE_GENERIC"] = old
        outs[name] = pcm
        pos = 0
        for s in range(S):
            n = want[s].shape[1]
            assert chains[s].status == 0 and chains[s].n_samples == n, (name, s)
            blk = pcm[pos: pos + n * channels]
            got = blk.reshape(n, channels).T if interleaved else blk.reshape(channels, n)
            if dt == np.float32:
                assert bits_equal(got, want[s]), (name, s, mismatch_report(got, want[s]))
            else:
                assert np.array_equal(got, oracle.quantise_i16(want[s])), (name, s)
            pos += n * channels
            assert bits_equal(pwrs[s].data(), refs[s].pwr.data()), (name, s)
    assert np.array_equal(outs["chain"].view(np.uint8), outs["four"].view(np.uint8))


# BASELINE.json configs[2]: 5.1 channels, 256/2048 mixed blocks, residue coupling chained through a shared channel
_COUPLING_51 = [(0, 1), (2, 3), (0, 4)]


def _mixed_variant_kernels(name, bs0, residue, memory):
    """expect_kernels arguments of one variant of test_mixed_streams_are_segmented_between_fused_and_chain_kernels: the
    kernels that variant exists to run, and the ones its switch disables."""
    if name == "chain":                                  # LWB_NO_MIXED: the chain kernel alone, its own front half
        return dict(ran={"k_chain"}, not_ran=ALL_KERNELS - {"k_chain"})
    not_ran = set(GENERIC) | {"k_mid"}
    ran = set(FRONT) if residue else set()
    if bs0 == 8 and name in ("mixed", "mixed_nobalance", "mixed_nobursts", "mixed_chunked"):
        ran |= {"k_long_s"}                              # the one-pass schedule
        if memory == cabi.MEM_DEVICE:
            not_ran |= {"k_long", "k_chain"}             # (no rounds behind it)
    else:                                                # rounds: k_long, and k_short (bs0 == 8) or k_chain for the rest
        ran |= {"k_long", "k_short" if bs0 == 8 and name != "mixed_noshort" else "k_chain"}
        not_ran |= {"k_long_s", "k_short_g", "k_row_copy"}
    if name == "mixed_nobursts":
        not_ran |= {"k_short_g"}
    if name == "mixed_noshort" or bs0 != 8:
        not_ran |= {"k_short", "k_short_g"}
    return dict(ran=ran, not_ran=not_ran)


@pytest.mark.parametrize("entry,memory,fmt,seed,bs0,channels", [
    ("spectrum", cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 80, 8, 2),
    ("spectrum", cabi.MEM_DEVICE, cabi.OUT_I16_PLANAR, 81, 8, 2),
    ("residue", cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 82, 8, 2),
    ("residue", cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 83, 8, 2),
    ("spectrum", cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 84, 6, 2),
    ("spectrum", cabi.MEM_HOST, cabi.OUT_I16_PLANAR, 85, 10, 2),
    ("residue", cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 86, 11, 2),
    # config 3 on the path that serves it: try_mixed -> batched k_prologue (8-way coupled-channel path)
    # -> k_long with transitional blocks -> k_chain, residue entry, planar f32 and i16, host and device
    ("residue", cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 87, 8, 6),
    ("residue", cabi.MEM_DEVICE, cabi.OUT_I16_PLANAR, 88, 8, 6),
    ("residue", cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 89, 8, 6),
    ("spectrum", cabi.MEM_HOST, cabi.OUT_I16_PLANAR, 90, 8, 6)])
def test_mixed_streams_are_segmented_between_fused_and_chain_kernels(ctx, oracle, entry, memory, fmt, seed, bs0, channels):
    """The standard 256/2048 stream shape: mostly long blocks with bursts of short ones.  The host cuts
    every chain into long-run segments (fused kernel) and the rest (chain kernel) and runs them round
    by round, handing PreviousWindowRight over through the device state.  Bit-exact against the oracle,
    over two consecutive batches (state carried across), and identical to the chain-kernel-only path.
    The 6-channel cases are BASELINE.json configs[2]: the coupling steps chain through channel 0
    (audio.rs:991-1002 applies them in reverse), window shapes per audio.rs:1059-1073."""
    rng = np.random.default_rng(seed)
    bs1, S, P = 11, 6, 40
    residue = entry == "residue"
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    if channels == 6:
        mappings[0]["coupling"] = list(_COUPLING_51)
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    outs = {}
    cases = []
    refs = [RefStream(oracle, channels, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    # one consistent sequence of 2P packets per stream, decoded as two batches of P
    full = [mode_sequence(rng, 2 * P, p_short=0.12 if s else 0.5) for s in range(S)]
    bf, prev, nxt = full[1]
    bf[P - 1:] = 1; prev[P:] = 1; nxt[P - 1:] = 1           # an all-long chain inside the second batch
    prev[P - 1] = bf[P - 2]
    if bf[P - 2]:
        nxt[P - 2] = 1
    for batch in range(2):
        coeffs, dense, kinds, ys, want, seqs = [], [], [], [], [], []
        for s in range(S):
            bf, prev, nxt = (a[batch * P:(batch + 1) * P] for a in full[s])
            mode_ids = np.array([int(rng.choice([m for m in range(4) if modes[m][0] == b])) for b in bf], np.uint8)
            parts = []
            for i in range(P):
                n2 = (1 << (bs1 if bf[i] else bs0)) // 2
                res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
                if residue:
                    mp = mappings[modes[mode_ids[i]][1]]
                    fl = []
                    for c in range(channels):
                        mult, xs = floors[mp["floor_of_channel"][c]]
                        r = rng.random()
                        fl.append(None if r < 0.1 else (rng.random(n2).astype(np.float32) if r < 0.2
                                                        else random_floor1_y(rng, mult, len(xs))))
                    rc, pcm = refs[s].packet(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res, fl)
                    k, y, d = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
                    dense.append((d if d is not None else np.zeros_like(res)).ravel())
                    kinds.append(k)
                    ys.append(y)
                else:
                    rc, pcm = refs[s].spectrum(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res)
                assert rc == 0
                parts.append(pcm)
                coeffs.append(res.ravel())
            want.append(np.concatenate(parts, axis=1))
            seqs.append((mode_ids, prev, nxt))
        cases.append((np.concatenate(coeffs), np.concatenate(dense) if residue else None,
                      np.concatenate(kinds) if residue else None, np.concatenate(ys) if residue else None, want, seqs,
                      [r.pwr.data().copy() for r in refs]))
    # "mixed": k_long + k_short (bs0 == 8) + k_chain rounds; "mixed_noshort": short blocks through the chain kernel
    # "mixed_rounds": segment by segment, the state handed over between launches (what batches that are not a strict
    # long / short alternation still do); "mixed" runs k_long once and k_short once when bs0 == 8
    variants = [("mixed", None), ("chain", {"LWB_NO_MIXED": "1"}), ("mixed_noshort", {"LWB_NO_SHORT": "1"}),
                ("mixed_rounds", {"LWB_MIXED_ROUNDS": "1"}),
                ("mixed_nobalance", {"LWB_NO_BALANCE": "1"}),       # the static deals in segment order
                ("mixed_nobursts", {"LWB_NO_BURSTS": "1"})]         # bursts through k_short (one octet each) instead of k_short_g
    if memory == cabi.MEM_HOST:
        variants.append(("mixed_chunked", {"LWB_E2E_CHUNKS": "3"}))       # H2D / kernels / D2H pipelined over 3 chunks of chains
    for name, env in variants:
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        for batch, (coeffs, dense, kinds, ys, want, seqs, end_state) in enumerate(cases):
            chains, coeff_off, out_off = [], 0, 0
            for s in range(S):
                n = want[s].shape[1]
                mode_ids, prev, nxt = seqs[s]
                chains.append(L.ChainSpec(pwrs[s], mode_ids, prev, nxt, coeff_offset=coeff_off, packet_index=s * P,
                                          out_offset=out_off, out_stride=n))
                coeff_off += sum(channels * ((1 << (bs1 if modes[m][0] else bs0)) // 2) for m in mode_ids)
                out_off += n * channels
            pcm = np.zeros(out_off, dt)
            if env:
                os.environ.update(env)
            launches0 = ctx.launch_count
            with expect_kernels(ctx, **_mixed_variant_kernels(name, bs0, residue, memory)) as launched:
                try:
                    kw = dict(floor_kind=kinds, floor1_y=ys, dense_floor=dense) if residue else {}
                    if memory == cabi.MEM_DEVICE:
                        d_in = ctx.device_alloc(coeffs.nbytes)
                        d_out = ctx.device_alloc(max(pcm.nbytes, 4))
                        ctx.h2d(d_in, coeffs)
                        if residue:
                            d_dense = ctx.device_alloc(dense.nbytes)
                            ctx.h2d(d_dense, dense)
                            kw["dense_floor"] = d_dense
                        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE if residue else cabi.ENTRY_SPECTRUM, memory, d_in, d_out, fmt, **kw)
                        ctx.d2h(pcm, d_out)
                        ctx.device_free(d_in)
                        ctx.device_free(d_out)
                        if residue:
                            ctx.device_free(d_dense)
                    else:
                        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE if residue else cabi.ENTRY_SPECTRUM, memory, coeffs, pcm, fmt, **kw)
                finally:
                    if env:
                        for k in env:
                            del os.environ[k]
                n_launch = ctx.launch_count - launches0
            one_pass = name in ("mixed", "mixed_nobalance", "mixed_nobursts") and bs0 == 8
            if one_pass:        # the pass's short segments: k_short (eight packets and more) and / or k_short_g (bursts)
                assert launched["k_short"] + launched["k_short_g"] >= 1, launched
            if one_pass and memory == cabi.MEM_DEVICE:
                # (two front stages +) k_long + k_short, no rounds; streams with history: their state rows are copied first
                # k_short takes the short runs of eight packets and more, k_short_g the bursts: one of them or both
                lo = (4 if residue else 2) + (1 if batch else 0)
                assert lo <= n_launch <= lo + 1, n_launch
            elif name.startswith("mixed"):
                assert n_launch >= (2 if one_pass else 3), n_launch      # fused + chain + fused/chain rounds
            else:
                assert n_launch == 1, n_launch
            outs[(name, batch)] = pcm
            pos = 0
            for s in range(S):
                n = want[s].shape[1]
                assert chains[s].status == 0 and chains[s].n_samples == n, (name, batch, s)
                got = pcm[pos: pos + n * channels].reshape(channels, n)
                if f32:
                    assert bits_equal(got, want[s]), (name, batch, s, mismatch_report(got, want[s]))
                else:
                    assert np.array_equal(got, oracle.quantise_i16(want[s])), (name, batch, s)
                pos += n * channels
                assert bits_equal(pwrs[s].data(), end_state[s]), (name, batch, s)
    for batch in range(2):
        for name, _ in variants[1:]:
            assert np.array_equal(outs[("mixed", batch)].view(np.uint8), outs[(name, batch)].view(np.uint8)), name


@pytest.mark.parametrize("bs,channels,fmt,memory,seed", [
    (10, 1, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 400), (10, 2, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 401),
    (10, 6, cabi.OUT_F32_PLANAR, cabi.MEM_HOST, 402), (10, 3, cabi.OUT_I16_PLANAR, cabi.MEM_DEVICE, 403),
    (9, 1, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 404), (9, 2, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 405),
    (9, 5, cabi.OUT_F32_PLANAR, cabi.MEM_HOST, 406), (9, 3, cabi.OUT_I16_PLANAR, cabi.MEM_DEVICE, 407)])
def test_mid_block_kernel_uniform_batches(ctx, oracle, bs, channels, fmt, memory, seed):
    """Uniform 1024- and 512-point streams (blocksize 10 / 9) through k_mid: two / four runs per warp in lockstep, so
    chains of different lengths exercise the grouping by length and the dummy partners of a short group, many chains the
    static deal with several groups per warp; three consecutive batches carry the state (none, then n/2 samples);
    bit-exact against the oracle and byte-identical to the chain kernel (LWB_NO_MID=1)."""
    n2 = 1 << (bs - 1)
    rng = np.random.default_rng(seed)
    S = 700 if channels == 1 else 257
    D = 5
    modes = [(1, 0)]
    su = make_setup(ctx, channels, bs, bs, modes=modes)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    lens = [int(rng.integers(1, 7)) for _ in range(D)]
    refs = [RefStream(oracle, channels, bs, bs, modes) for _ in range(D)]
    outs = {}
    batches = []
    for b in range(3):
        specs = [rng.standard_normal((lens[d], channels, n2)).astype(np.float32) for d in range(D)]
        want = []
        for d in range(D):
            parts = []
            for i in range(lens[d]):
                rc, pcm = refs[d].spectrum(0, 1, 1, specs[d][i])
                assert rc == 0
                parts.append(pcm)
            want.append((np.concatenate(parts, axis=1), refs[d].pwr.data().copy()))
        batches.append((specs, want))
    for name, env in (("mid", None), ("chain", {"LWB_NO_MID": "1"})):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        if env:
            os.environ.update(env)
        try:
            for b, (specs, want) in enumerate(batches):
                chains, coeffs, coeff_off, out_off = [], [], 0, 0
                for s in range(S):
                    d = s % D
                    stride = lens[d] * n2
                    chains.append(L.ChainSpec(pwrs[s], np.zeros(lens[d], np.uint8), coeff_offset=coeff_off, out_offset=out_off,
                                              out_stride=stride))
                    coeffs.append(specs[d].ravel())
                    coeff_off += specs[d].size
                    out_off += stride * channels
                coeffs = np.concatenate(coeffs)
                pcm = np.zeros(out_off, dt)
                k = "k_mid" if name == "mid" else "k_chain"
                with expect_kernels(ctx, ran={k: 1}, not_ran=ALL_KERNELS - {k}):
                    if memory == cabi.MEM_DEVICE:
                        d_in, d_out = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
                        ctx.h2d(d_in, coeffs)
                        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, d_in, d_out, fmt)
                        ctx.d2h(pcm, d_out)
                        ctx.device_free(d_in)
                        ctx.device_free(d_out)
                    else:
                        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, coeffs, pcm, fmt)
                pos = 0
                got_all = []
                for s in range(S):
                    d = s % D
                    stride = lens[d] * n2
                    n = want[d][0].shape[1]
                    assert chains[s].status == 0 and chains[s].n_samples == n, (name, b, s)
                    got = pcm[pos: pos + stride * channels].reshape(channels, stride)[:, :n]
                    if f32:
                        assert bits_equal(got, want[d][0]), (name, b, s, mismatch_report(got, want[d][0]))
                    else:
                        assert np.array_equal(got, oracle.quantise_i16(want[d][0])), (name, b, s)
                    got_all.append(got.copy())
                    pos += stride * channels
                for s in range(0, S, 41):
                    assert bits_equal(pwrs[s].data(), want[s % D][1]), (name, b, s)
                outs[(name, b)] = got_all
        finally:
            if env:
                for k in env:
                    del os.environ[k]
    for b in range(3):
        for s in range(S):
            assert np.array_equal(outs[("mid", b)][s].view(np.uint8), outs[("chain", b)][s].view(np.uint8)), (b, s)


@pytest.mark.parametrize("fmt,seed,p_bad", [(cabi.OUT_F32_PLANAR, 300, 0.0), (cabi.OUT_I16_PLANAR, 301, 0.0),
                                            (cabi.OUT_F32_PLANAR, 302, 0.08), (cabi.OUT_I16_PLANAR, 303, 0.3),
                                            (cabi.OUT_F32_PLANAR, 304, 0.004), (cabi.OUT_I16_PLANAR, 305, 0.01)])
def test_segmented_paths_agree_with_chain_kernel_on_arbitrary_flags(ctx, fmt, seed, p_bad):
    """Differential: whatever the caller passes as previous / next window flags -- consistent with the neighbouring
    packets or not -- and wherever a chain stops on a bad mode number, the segmented schedules (one pass where every
    chain alternates cleanly between long and short segments, rounds as soon as one does not) must produce the same
    bytes, statuses, sample counts and end states as the chain kernel alone.  p_bad = 0: consistent flags (all chains
    take the one-pass schedule); otherwise that share of the flags is flipped and a few mode numbers are invalid (0.004 /
    0.01: most chains stay clean and take the pass, the others run their rounds behind it).
    Three consecutive batches, so every schedule starts from every kind of state the others left."""
    rng = np.random.default_rng(seed)
    S, P, C = 96, 20, 2
    modes = [(0, 0), (1, 0)]
    su = make_setup(ctx, C, 8, 11, modes=modes)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    batches = []
    for b in range(3):
        seqs = []
        for s in range(S):
            bf, prev, nxt = mode_sequence(rng, P, p_short=float(rng.choice([0.1, 0.3, 0.6])))
            mode_ids = bf.astype(np.uint8)
            if p_bad:
                flip = rng.random(P) < p_bad
                prev = np.where(flip, 1 - prev, prev).astype(np.uint8)
                flip = rng.random(P) < p_bad
                nxt = np.where(flip, 1 - nxt, nxt).astype(np.uint8)
                if rng.random() < 0.2:
                    mode_ids[int(rng.integers(0, P))] = 7             # no such mode: the chain stops there
            seqs.append((mode_ids, prev, nxt))
        n_coeff = sum(int(sum(C * (1024 if m == 1 else 128) for m in sq[0])) for sq in seqs)
        batches.append((seqs, (rng.standard_normal(n_coeff) * 0.1).astype(np.float32)))
    results = {}
    for name, env in (("segmented", None), ("rounds", {"LWB_MIXED_ROUNDS": "1"}), ("chain", {"LWB_NO_MIXED": "1"})):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        log = []
        launches0 = ctx.launch_count
        # LWB_MIXED_ROUNDS turns the one pass (k_long_s) off, LWB_NO_MIXED the fused kernels
        off = {"segmented": set(), "rounds": {"k_long_s", "k_short_g", "k_row_copy"}, "chain": ALL_KERNELS - {"k_chain"}}[name]
        with expect_kernels(ctx, ran={"segmented": {"k_long_s"} if not p_bad else set(), "rounds": {"k_long"},
                                      "chain": {"k_chain"}}[name], not_ran=off | GENERIC):
            if env:
                os.environ.update(env)
            try:
                for seqs, coeffs in batches:
                    chains, coeff_off = [], 0
                    stride = P * 1536          # (a long block in front of a short one emits up to 1472 samples)
                    for s in range(S):
                        mode_ids, prev, nxt = seqs[s]
                        chains.append(L.ChainSpec(pwrs[s], mode_ids, prev, nxt, coeff_offset=coeff_off, out_offset=s * C * stride,
                                                  out_stride=stride))
                        coeff_off += int(sum(C * (1024 if m == 1 else 128) for m in mode_ids))
                    pcm = np.zeros(S * C * stride, dt)
                    L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, coeffs, pcm, fmt)
                    rows = pcm.reshape(S, C, stride)
                    log.append(([(c.status, c.n_samples, c.packets_done) for c in chains],
                                [rows[s, :, :chains[s].n_samples].copy() for s in range(S)],
                                [None if p.is_empty() else p.data().copy() for p in pwrs]))
            finally:
                if env:
                    for k in env:
                        del os.environ[k]
        results[name] = log
        results[name + "_launches"] = ctx.launch_count - launches0
    # clean chains take the one pass (when they are the larger part of the batch), the others their rounds behind it
    if not p_bad:       # (batches 1 and 2 start some chains on a state their first packet's flags contradict: those keep rounds)
        assert results["segmented_launches"] < results["rounds_launches"], (results["segmented_launches"], results["rounds_launches"])
    for name in ("segmented", "rounds"):
        for b in range(3):
            st_a, pcm_a, pw_a = results[name][b]
            st_c, pcm_c, pw_c = results["chain"][b]
            assert st_a == st_c, (name, b)
            for s in range(S):
                assert np.array_equal(pcm_a[s].view(np.uint8), pcm_c[s].view(np.uint8)), (name, b, s)
                assert (pw_a[s] is None) == (pw_c[s] is None), (name, b, s)
                assert pw_a[s] is None or bits_equal(pw_a[s], pw_c[s]), (name, b, s)
    if not p_bad:
        assert all(st == 0 for st, _, _ in results["segmented"][0][0])


@pytest.mark.parametrize("fmt,bursts,p_short", [(cabi.OUT_F32_PLANAR, True, 0.3), (cabi.OUT_I16_PLANAR, True, 0.5),
                                               (cabi.OUT_F32_PLANAR, False, 0.3), (cabi.OUT_F32_PLANAR, True, 0.08)])
def test_one_pass_schedule_many_runs_per_warp(ctx, oracle, fmt, bursts, p_short):
    """The one-pass schedule of mixed streams at scale: thousands of chains, so every warp of k_long_s and of
    k_short_g (bursts=False: k_short) walks dozens of one- to three-packet runs, its prefetch (tiles, descriptors, state rows) crossing many run
    boundaries, every boundary handing 128 samples over through a slot.  Two consecutive batches: the second starts
    from stream state, which the pass moves out of the way first (k_row_copy).  The chains repeat 6 distinct streams,
    so the oracle decodes 6 and the comparison covers all."""
    rng = np.random.default_rng(int(p_short * 100) + (0 if bursts else 7))
    S, D, P, C = 2000, 6, 24, 2
    modes = [(0, 0), (1, 0)]
    su = make_setup(ctx, C, 8, 11, modes=modes)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    seqs = [mode_sequence(rng, 2 * P, p_short=p_short) for _ in range(D)]
    refs = [RefStream(oracle, C, 8, 11, modes) for _ in range(D)]
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    if not bursts:
        os.environ["LWB_NO_BURSTS"] = "1"
    try:
        for batch in range(2):
            want, specs, states = [], [], []
            for d in range(D):
                bf, prev, nxt = (a[batch * P:(batch + 1) * P] for a in seqs[d])
                parts, sp = [], []
                for i in range(P):
                    res = rng.standard_normal((C, 1024 if bf[i] else 128)).astype(np.float32)
                    rc, pcm = refs[d].spectrum(int(bf[i]), int(prev[i]), int(nxt[i]), res)
                    assert rc == 0
                    parts.append(pcm)
                    sp.append(res.ravel())
                want.append(np.concatenate(parts, axis=1))
                specs.append(np.concatenate(sp))
                states.append(refs[d].pwr.data().copy())
            chains, coeffs, coeff_off, out_off = [], [], 0, 0
            for s in range(S):
                d = s % D
                bf, prev, nxt = (a[batch * P:(batch + 1) * P] for a in seqs[d])
                n = want[d].shape[1]
                chains.append(L.ChainSpec(pwrs[s], bf.astype(np.uint8), prev, nxt, coeff_offset=coeff_off, out_offset=out_off,
                                          out_stride=n))
                coeffs.append(specs[d])
                coeff_off += specs[d].size
                out_off += n * C
            coeffs = np.concatenate(coeffs)
            pcm = np.zeros(out_off, dt)
            launches0 = ctx.launch_count
            # the one pass: k_long_s, then k_short_g over the bursts (LWB_NO_BURSTS: k_short takes them), k_row_copy once
            # there is state to move
            ran = {"k_long_s", "k_short_g" if bursts else "k_short"} | ({"k_row_copy"} if batch else set())
            with expect_kernels(ctx, ran=ran, not_ran=GENERIC | {"k_long", "k_chain", "k_mid"} | (set() if bursts else {"k_short_g"})):
                L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, coeffs, pcm, fmt)
            assert ctx.launch_count - launches0 <= 4 * 8, ctx.launch_count - launches0      # (copy +) k_long_s + k_short (+ k_short_g) per host chunk
            pos = 0
            for s in range(S):
                d = s % D
                n = want[d].shape[1]
                assert chains[s].status == 0 and chains[s].n_samples == n, (batch, s)
                got = pcm[pos: pos + n * C].reshape(C, n)
                if f32:
                    assert bits_equal(got, want[d]), (batch, s, mismatch_report(got, want[d]))
                else:
                    assert np.array_equal(got, oracle.quantise_i16(want[d])), (batch, s)
                pos += n * C
            for s in range(0, S, 97):
                assert bits_equal(pwrs[s].data(), states[s % D]), (batch, s)
    finally:
        os.environ.pop("LWB_NO_BURSTS", None)


@pytest.mark.parametrize("P", [1, 2, 3, 5, 6])
def test_fused_kernel_many_short_runs_per_warp(ctx, oracle, P):
    """More runs than warps, each shorter than (or as long as) the kernel's tile ring: every warp walks
    several groups and its prefetch crosses several run boundaries.  All chains carry the same few
    distinct inputs, so the oracle decodes 7 streams and the comparison covers all of them."""
    rng = np.random.default_rng(90 + P)
    S, D = 6000, 7
    su = make_setup(ctx, 1, 8, 11)
    spec_d = rng.standard_normal((D, P, 1024)).astype(np.float32)
    want = []
    for d in range(D):
        ref = RefStream(oracle, 1, 8, 11, [(0, 0), (1, 0)])
        parts = []
        for i in range(P):
            rc, pcm = ref.spectrum(1, 1, 1, spec_d[d, i][None])
            assert rc == 0
            parts.append(pcm)
        want.append((np.concatenate(parts, axis=1), ref.pwr.data().copy()))
    n = want[0][0].shape[1]
    spec = np.ascontiguousarray(spec_d[np.arange(S) % D]).ravel()
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    modes = np.ones(P, np.uint8)
    stride = max(n, 4)
    chains = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * 1024, out_offset=s * stride, out_stride=stride) for s in range(S)]
    pcm = np.full(S * stride, np.nan, np.float32)
    launches0 = ctx.launch_count
    with expect_kernels(ctx, **long_batch_kernels(None)):
        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, spec, pcm, cabi.OUT_F32_PLANAR)
    assert ctx.launch_count - launches0 <= 8            # fused kernel (one launch per host chunk)
    got = pcm.reshape(S, stride)[:, :n]
    for s in range(S):
        assert chains[s].status == 0 and chains[s].n_samples == n
    for d in range(D):
        blk = got[d::D]
        assert np.array_equal(blk.view(np.uint32), np.broadcast_to(want[d][0].view(np.uint32), blk.shape)), d
    for s in (0, 1, S // 2, S - 1):
        assert bits_equal(pwrs[s].data(), want[s % D][1])
    # second batch on top of the saved state
    want2 = []
    for d in range(D):
        ref = RefStream(oracle, 1, 8, 11, [(0, 0), (1, 0)])
        parts = []
        for rep in range(2):
            for i in range(P):
                rc, o = ref.spectrum(1, 1, 1, spec_d[d, i][None])
                if rep:
                    parts.append(o)
        want2.append(np.concatenate(parts, axis=1))
    n2 = want2[0].shape[1]
    pcm2 = np.full(S * P * 1024, np.nan, np.float32)
    chains2 = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * 1024, out_offset=s * P * 1024, out_stride=P * 1024) for s in range(S)]
    with expect_kernels(ctx, **long_batch_kernels(None)):
        L.decode_chains(ctx, chains2, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, spec, pcm2, cabi.OUT_F32_PLANAR)
    got2 = pcm2.reshape(S, P * 1024)[:, :n2]
    assert n2 == P * 1024
    for d in range(D):
        blk = got2[d::D]
        assert np.array_equal(blk.view(np.uint32), np.broadcast_to(want2[d].view(np.uint32), blk.shape)), d
    for p_ in pwrs:
        p_.close()


@pytest.mark.parametrize("bs,channels,fmt,memory,seed", [(10, 2, cabi.OUT_F32_PLANAR, cabi.MEM_HOST, 420), (10, 6, cabi.OUT_I16_PLANAR, cabi.MEM_DEVICE, 421),
                                                         (9, 2, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 422), (9, 3, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 423)])
def test_mid_block_kernel_residue_entry(ctx, oracle, bs, channels, fmt, memory, seed):
    """Residue entry in front of k_mid: full packets (coupling, floor-1 / dense / unused floors) of uniform 1024- / 512-point
    streams: k_floor1_segments + k_prologue_fused form the spectrum, k_mid transforms it; bit-exact against the oracle over
    two batches and byte-identical to the chain kernel (LWB_NO_MID=1), which does the same work inside one kernel."""
    rng = np.random.default_rng(seed)
    S, P = 9, 4
    n2 = 1 << (bs - 1)
    floors, mappings, modes = _random_packet_case(rng, channels, bs, bs)
    su = make_setup(ctx, channels, bs, bs, modes=modes, mappings=mappings, floors=floors)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    refs = [RefStream(oracle, channels, bs, bs, modes, mappings, floors) for _ in range(S)]
    batches = []
    for b in range(2):
        coeffs, dense, kinds, ys, want, seqs, raw = [], [], [], [], [], [], []
        for s in range(S):
            mode_ids = rng.integers(0, len(modes), P).astype(np.uint8)
            parts = []
            raw.append([])
            for i in range(P):
                res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
                mp = mappings[modes[mode_ids[i]][1]]
                fl = []
                for c in range(channels):
                    mult, xs = floors[mp["floor_of_channel"][c]]
                    r = rng.random()
                    fl.append(None if r < 0.15 else (rng.random(n2).astype(np.float32) if r < 0.25 else random_floor1_y(rng, mult, len(xs))))
                rc, pcm = refs[s].packet(int(mode_ids[i]), 1, 1, res, fl)
                assert rc == 0
                parts.append(pcm)
                raw[-1].append((int(mode_ids[i]), res, fl))
                k, y, d = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
                coeffs.append(res.ravel())
                dense.append((d if d is not None else np.zeros_like(res)).ravel())
                kinds.append(k)
                ys.append(y)
            want.append(np.concatenate(parts, axis=1))
            seqs.append(mode_ids)
        batches.append((np.concatenate(coeffs), np.concatenate(dense), np.concatenate(kinds), np.concatenate(ys), want, seqs,
                        [r.pwr.data().copy() for r in refs], raw))
    outs = {}
    for name, env in (("mid", None), ("chain", {"LWB_NO_MID": "1"})):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        if env:
            os.environ.update(env)
        try:
            for b, (coeffs, dense, kinds, ys, want, seqs, end_state, _raw) in enumerate(batches):
                stride = P * n2
                chains = [L.ChainSpec(pwrs[s], seqs[s], coeff_offset=s * P * channels * n2, packet_index=s * P,
                                      out_offset=s * channels * stride, out_stride=stride) for s in range(S)]
                pcm = fill_guard(np.empty(S * channels * stride, dt))
                launches0 = ctx.launch_count
                # mid: the front stages, then k_mid; LWB_NO_MID: the chain kernel with its own front half
                want_k = {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_mid": 1} if name == "mid" else {"k_chain": 1}
                with expect_kernels(ctx, ran=want_k, not_ran=ALL_KERNELS - set(want_k)):
                    if memory == cabi.MEM_DEVICE:
                        d_in, d_out, d_dense = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(pcm.nbytes), ctx.device_alloc(dense.nbytes)
                        ctx.h2d(d_in, coeffs)
                        ctx.h2d(d_dense, dense)
                        ctx.h2d(d_out, pcm)
                        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, d_in, d_out, fmt, floor_kind=kinds, floor1_y=ys, dense_floor=d_dense)
                        ctx.d2h(pcm, d_out)
                        for h in (d_in, d_out, d_dense):
                            ctx.device_free(h)
                    else:
                        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, coeffs, pcm, fmt, floor_kind=kinds, floor1_y=ys, dense_floor=dense)
                assert ctx.launch_count - launches0 == (3 if name == "mid" else 1)
                for s in range(S):
                    n = want[s].shape[1]
                    assert chains[s].status == 0 and chains[s].n_samples == n, (name, b, s)
                    got = pcm[s * channels * stride: (s + 1) * channels * stride].reshape(channels, stride)[:, :n]
                    if f32:
                        assert bits_equal(got, want[s]), (name, b, s, mismatch_report(got, want[s]))
                    else:
                        assert np.array_equal(got, oracle.quantise_i16(want[s])), (name, b, s)
                    assert bits_equal(pwrs[s].data(), end_state[s]), (name, b, s)
                assert_contained(pcm, write_set(chains, lambda i: channels, fmt), (name, b))
                outs[(name, b)] = pcm
        finally:
            if env:
                for k in env:
                    del os.environ[k]
    for b in range(2):
        assert np.array_equal(outs[("mid", b)].view(np.uint8), outs[("chain", b)].view(np.uint8)), b
    if memory == cabi.MEM_DEVICE:
        # a prepared batch: plans, re-plans once the streams hold state, then replays front stages + k_mid from the plan
        coeffs, dense, kinds, ys, _want, seqs, _end, raw = batches[0]
        refs2 = [RefStream(oracle, channels, bs, bs, modes, mappings, floors) for _ in range(S)]
        pwrs2 = [L.PreviousWindowRight(su) for _ in range(S)]
        stride = P * n2
        chains = [L.ChainSpec(pwrs2[s], seqs[s], coeff_offset=s * P * channels * n2, packet_index=s * P,
                              out_offset=s * channels * stride, out_stride=stride) for s in range(S)]
        d_in, d_dense = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(dense.nbytes)
        d_out = ctx.device_alloc(S * channels * stride * dt().itemsize)
        ctx.h2d(d_in, coeffs)
        ctx.h2d(d_dense, dense)
        batch = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, d_in, d_out, fmt, floor_kind=kinds, floor1_y=ys, dense_floor=d_dense)
        for it in range(4):
            pcm = np.zeros(S * channels * stride, dt)
            with expect_kernels(ctx, ran={"k_floor1_segments": 1, "k_prologue_fused": 1, "k_mid": 1},
                                not_ran=ALL_KERNELS - FRONT - {"k_mid"}):
                batch.run()
            ctx.synchronize()
            ctx.d2h(pcm, d_out)
            batch.collect()
            for s in range(S):
                parts = []
                for mode, res, fl in raw[s]:
                    rc, o = refs2[s].packet(mode, 1, 1, res, fl)
                    assert rc == 0
                    parts.append(o)
                w = np.concatenate(parts, axis=1)
                n = w.shape[1]
                assert chains[s].status == 0 and chains[s].n_samples == n, (it, s)
                got = pcm[s * channels * stride: (s + 1) * channels * stride].reshape(channels, stride)[:, :n]
                if f32:
                    assert bits_equal(got, w), ("plan", it, s, mismatch_report(got, w))
                else:
                    assert np.array_equal(got, oracle.quantise_i16(w)), ("plan", it, s)
        batch.close()
        for h in (d_in, d_dense, d_out):
            ctx.device_free(h)


@pytest.mark.parametrize("bs", [10, 9])
def test_prepared_mid_batch_replays(ctx, oracle, bs):
    """A prepared batch of uniform 1024- / 512-point chains in device memory (k_mid): the first execution plans and runs,
    the second re-plans (the streams now hold state), later ones replay the captured launch.  Every execution is checked
    against the oracle, which decodes the same packets again on top of its own state."""
    rng = np.random.default_rng(500 + bs)
    channels, S, P = 2, 37, 5
    n2 = 1 << (bs - 1)
    modes = [(1, 0)]
    su = make_setup(ctx, channels, bs, bs, modes=modes)
    refs = [RefStream(oracle, channels, bs, bs, modes) for _ in range(S)]
    specs = rng.standard_normal((S, P, channels, n2)).astype(np.float32)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    stride = P * n2
    chains = [L.ChainSpec(pwrs[s], np.zeros(P, np.uint8), coeff_offset=s * P * channels * n2, out_offset=s * channels * stride,
                          out_stride=stride) for s in range(S)]
    d_in = ctx.device_alloc(specs.nbytes)
    d_out = ctx.device_alloc(S * channels * stride * 4)
    ctx.h2d(d_in, specs.ravel())
    batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, d_in, d_out, cabi.OUT_F32_PLANAR)
    for it in range(4):
        pcm = np.full(S * channels * stride, np.nan, np.float32)
        ctx.h2d(d_out, pcm)
        with expect_kernels(ctx, ran={"k_mid": 1}, not_ran=ALL_KERNELS - {"k_mid"}):
            batch.run()
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        batch.collect()
        for s in range(S):
            parts = []
            for i in range(P):
                rc, o = refs[s].spectrum(0, 1, 1, specs[s, i])
                assert rc == 0
                parts.append(o)
            want = np.concatenate(parts, axis=1)
            n = want.shape[1]
            assert chains[s].status == 0 and chains[s].n_samples == n, (it, s)
            got = pcm[s * channels * stride: (s + 1) * channels * stride].reshape(channels, stride)[:, :n]
            assert bits_equal(got, want), (it, s, mismatch_report(got, want))
    for s in range(0, S, 7):
        assert bits_equal(pwrs[s].data(), refs[s].pwr.data()), s
    batch.close()
    ctx.device_free(d_in)
    ctx.device_free(d_out)


def test_prepared_mixed_batch_replays_captured_rounds(ctx, oracle):
    """A prepared batch of mixed short/long chains in device memory: the first execution plans and
    runs, the second re-plans (the streams now hold state), later ones replay the captured launch
    sequence without host planning.  Every execution is checked against the oracle, which decodes
    the same packets again on top of its own state."""
    rng = np.random.default_rng(95)
    channels, bs0, bs1, S, P = 2, 8, 11, 5, 30
    su = make_setup(ctx, channels, bs0, bs1)
    refs = [RefStream(oracle, channels, bs0, bs1, [(0, 0), (1, 0)]) for _ in range(S)]
    seqs, specs = [], []
    for s in range(S):
        bf = (rng.random(P) >= 0.15).astype(np.uint8)
        bf[0] = bf[-1] = 1                        # the sequence is decoded repeatedly: it must close on itself
        prev, nxt = np.ones(P, np.uint8), np.ones(P, np.uint8)
        for i in range(P):
            if bf[i]:
                prev[i] = bf[i - 1] if i else 1
                nxt[i] = bf[i + 1] if i + 1 < P else 1
        seqs.append((bf, prev, nxt))
        specs.append([rng.standard_normal((channels, 1024 if b else 128)).astype(np.float32) for b in bf])
    spec = np.concatenate([x.ravel() for sp in specs for x in sp])
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    stride = P * 1024
    chains, coeff_off = [], 0
    for s in range(S):
        chains.append(L.ChainSpec(pwrs[s], seqs[s][0], seqs[s][1], seqs[s][2], coeff_offset=coeff_off,
                                  out_offset=s * channels * stride, out_stride=stride))
        coeff_off += sum(x.size for x in specs[s])
    d_in = ctx.device_alloc(spec.nbytes)
    d_out = ctx.device_alloc(S * channels * stride * 4)
    ctx.h2d(d_in, spec)
    batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, d_in, d_out, cabi.OUT_F32_PLANAR)
    counts, kernels = [], []
    for it in range(4):
        pcm = np.full(S * channels * stride, np.nan, np.float32)
        ctx.h2d(d_out, pcm)
        l0 = ctx.launch_count
        with expect_kernels(ctx, ran={"k_long_s"}, not_ran=GENERIC | {"k_mid", "k_long"}) as launched:
            batch.run()
        kernels.append(launched)
        counts.append(ctx.launch_count - l0)
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        batch.collect()
        for s in range(S):
            parts = []
            for i in range(P):
                rc, o = refs[s].spectrum(int(seqs[s][0][i]), int(seqs[s][1][i]), int(seqs[s][2][i]), specs[s][i])
                assert rc == 0
                parts.append(o)
            want = np.concatenate(parts, axis=1)
            n = want.shape[1]
            assert chains[s].status == 0 and chains[s].n_samples == n, (it, s)
            got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, :n]
            assert bits_equal(got, want), (it, s, mismatch_report(got, want))
            assert bits_equal(pwrs[s].data(), refs[s].pwr.data()), (it, s)
    assert counts[1] == counts[2] == counts[3] and counts[1] >= 3, counts
    assert kernels[1] == kernels[2] == kernels[3], kernels       # a replay launches what the capturing execution did
    batch.close()
    ctx.device_free(d_in)
    ctx.device_free(d_out)


@pytest.mark.parametrize("shape,channels,fmt,floor_mem,seed", [
    ("long", 2, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 120),
    ("long", 2, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 121),
    ("long", 1, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 122),
    ("mixed", 6, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 123),
    ("mixed", 2, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 124),
    ("mixed", 6, cabi.OUT_I16_PLANAR, cabi.MEM_DEVICE, 125)])
def test_prepared_residue_batches_replay_front_stages(ctx, oracle, shape, channels, fmt, floor_mem, seed):
    """Residue-entry prepared batches in device memory (what a decode server replays step after step): the
    front stages (k_floor1_segments + k_prologue_fused: audio.rs:391-555, :991-1039) and the kernels behind them are
    captured once and replayed with NEW residues and floor posts every step -- from device-resident floor arrays
    (lwb_batch_io::floor_memory = LWB_MEM_DEVICE, read in place) or host arrays (uploaded again per step).
    "long": uniform long blocks (front stages + fused kernel); "mixed": 256/2048 sequences incl. the 5.1 coupling
    chain of BASELINE.json configs[2] (front stages + segmented k_long / k_chain rounds).  Every step is compared
    with the oracle, which keeps decoding on top of its own state."""
    rng = np.random.default_rng(seed)
    bs0, bs1, S, P = 8, 11, 5, 14 if shape == "long" else 26
    floors, mappings, modes = _random_packet_case(rng, channels, bs0, bs1)
    if channels == 6:
        mappings[0]["coupling"] = list(_COUPLING_51)
    elif channels == 2:
        mappings[0]["coupling"] = [(1, 0)] if seed % 2 else [(0, 1)]
    su = make_setup(ctx, channels, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    refs = [RefStream(oracle, channels, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    seqs = []
    for s in range(S):
        if shape == "long":
            bf = np.ones(P, np.uint8)
        else:
            bf = (rng.random(P) >= 0.2).astype(np.uint8)
            bf[0] = bf[-1] = 1                     # decoded repeatedly: the sequence must close on itself
        prev, nxt = np.ones(P, np.uint8), np.ones(P, np.uint8)
        for i in range(P):
            if bf[i]:
                prev[i] = bf[i - 1] if i else 1
                nxt[i] = bf[i + 1] if i + 1 < P else 1
        mode_ids = np.array([int(rng.choice([m for m in range(4) if modes[m][0] == b])) for b in bf], np.uint8)
        seqs.append((bf, prev, nxt, mode_ids))
    sizes = [[channels * (1024 if b else 128) for b in seqs[s][0]] for s in range(S)]
    total = sum(sum(x) for x in sizes)
    stride = P * 1024
    f32 = fmt == cabi.OUT_F32_PLANAR
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    chains, coeff_off = [], 0
    for s in range(S):
        chains.append(L.ChainSpec(pwrs[s], seqs[s][3], seqs[s][1], seqs[s][2], coeff_offset=coeff_off, packet_index=s * P,
                                  out_offset=s * channels * stride, out_stride=stride))
        coeff_off += sum(sizes[s])
    d_in = ctx.device_alloc(total * 4)
    d_out = ctx.device_alloc(S * channels * stride * 4)
    kinds = np.zeros((S * P, channels), np.uint8)
    ys = np.zeros((S * P, channels, cabi.MAX_POSTS), np.uint32)
    if floor_mem == cabi.MEM_DEVICE:
        d_kinds, d_ys = ctx.device_alloc(kinds.nbytes), ctx.device_alloc(ys.nbytes)
        batch = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, d_in, d_out, fmt, floor_kind=d_kinds, floor1_y=d_ys,
                        floor_memory=cabi.MEM_DEVICE)
    else:
        batch = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, d_in, d_out, fmt, floor_kind=kinds, floor1_y=ys)
    counts, kernels = [], []
    for it in range(4):
        coeffs, want = [], []
        for s in range(S):
            bf, prev, nxt, mode_ids = seqs[s]
            parts = []
            for i in range(P):
                n2 = 1024 if bf[i] else 128
                res = (rng.standard_normal((channels, n2)) * rng.integers(0, 2, (channels, n2))).astype(np.float32)
                mp = mappings[modes[mode_ids[i]][1]]
                fl = []
                for c in range(channels):
                    mult, xs = floors[mp["floor_of_channel"][c]]
                    fl.append(None if rng.random() < 0.1 else random_floor1_y(rng, mult, len(xs)))
                rc, o = refs[s].packet(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res, fl)
                assert rc == 0
                k, y, _ = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
                kinds[s * P + i], ys[s * P + i] = k, y
                parts.append(o)
                coeffs.append(res.ravel())
            want.append(np.concatenate(parts, axis=1))
        ctx.h2d(d_in, np.concatenate(coeffs))
        if floor_mem == cabi.MEM_DEVICE:
            ctx.h2d(d_kinds, kinds)
            ctx.h2d(d_ys, ys)
        pcm = np.zeros(S * channels * stride, np.float32 if f32 else np.int16)
        ctx.h2d(d_out, pcm)
        l0 = ctx.launch_count
        if shape == "long":
            ran, not_ran = {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_long": 1}, ALL_KERNELS - FRONT - {"k_long"}
        else:
            ran, not_ran = FRONT | {"k_long_s"}, GENERIC | {"k_mid"}
        with expect_kernels(ctx, ran=ran, not_ran=not_ran) as launched:
            batch.run()
        kernels.append(launched)
        counts.append(ctx.launch_count - l0)
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        batch.collect()
        for s in range(S):
            n = want[s].shape[1]
            assert chains[s].status == 0 and chains[s].n_samples == n, (it, s, chains[s].status, chains[s].n_samples, n)
            got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, :n]
            if f32:
                assert bits_equal(got, want[s]), (it, s, mismatch_report(got, want[s]))
            else:
                assert np.array_equal(got, oracle.quantise_i16(want[s])), (it, s)
            assert bits_equal(pwrs[s].data(), refs[s].pwr.data()), (it, s)
    assert counts[2] == counts[3], counts
    assert kernels[1] == kernels[2] == kernels[3], kernels       # step 1 captures, steps 2 and 3 replay: the same kernels
    if shape == "long":
        assert counts[3] == 3, counts              # k_floor1_segments + k_prologue_fused + k_long, nothing else
    batch.close()
    ctx.device_free(d_in)
    ctx.device_free(d_out)
    if floor_mem == cabi.MEM_DEVICE:
        ctx.device_free(d_kinds)
        ctx.device_free(d_ys)


@pytest.mark.parametrize("channels,P,S,fmt,memory,seed,sweep_setup", [
    (1, 8, 40, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 200, True),      # the n = 256 sweep shape: bs0 == bs1 == 8, one octet per run
    (2, 1, 7, cabi.OUT_F32_PLANAR, cabi.MEM_HOST, 201, False),
    (2, 3, 9, cabi.OUT_I16_PLANAR, cabi.MEM_DEVICE, 202, False),
    (6, 9, 5, cabi.OUT_F32_PLANAR, cabi.MEM_HOST, 203, False),
    (1, 131, 3, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 204, False),    # few long chains: runs are cut (primer packets)
    (2, 40, 300, cabi.OUT_I16_PLANAR, cabi.MEM_HOST, 205, False),     # more runs than warps: several runs per warp, ring crosses run boundaries
    (3, 17, 2, cabi.OUT_F32_PLANAR, cabi.MEM_DEVICE, 206, True)])
def test_short_block_kernel_uniform_batches(ctx, oracle, channels, P, S, fmt, memory, seed, sweep_setup):
    """Chains of 256-point blocks only (BASELINE.json configs[0] / configs[4] shapes) through lwb_decode_chains:
    the segmented path hands them to k_short (eight consecutive packets per warp step, imdct.rs:291-659 for
    n = 256 + audio.rs:1079-1154).  Three consecutive batches -- empty state, carried state, carried state -- bit-exact
    against the oracle and identical to the chain kernel; the state is compared after every batch."""
    rng = np.random.default_rng(seed)
    bs0, bs1 = (8, 8) if sweep_setup else (8, 11)
    modes = [(1, 0)] if sweep_setup else [(0, 0), (1, 0)]
    su = make_setup(ctx, channels, bs0, bs1, modes=modes)
    D = min(S, 6)                                   # distinct inputs: the oracle decodes D streams, the GPU all S
    refs = [RefStream(oracle, channels, bs0, bs1, modes) for _ in range(D)]
    f32 = fmt == cabi.OUT_F32_PLANAR
    outs = {}
    for name, env in (("short", None), ("chain", {"LWB_NO_SHORT": "1"})):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        rng_b = np.random.default_rng(seed + 1000)
        if name == "chain":
            refs = [RefStream(oracle, channels, bs0, bs1, modes) for _ in range(D)]
        for batch in range(3):
            spec_d = (rng_b.standard_normal((D, P, channels, 128)) * (1.0 if batch else 0.05)).astype(np.float32)
            want = []
            for d in range(D):
                parts = []
                for i in range(P):
                    rc, o = refs[d].spectrum(0, 1, 1, spec_d[d, i])
                    assert rc == 0
                    parts.append(o)
                want.append(np.concatenate(parts, axis=1))
            n = want[0].shape[1]
            spec = np.ascontiguousarray(spec_d[np.arange(S) % D]).ravel()
            stride = P * 128
            chains = [L.ChainSpec(pwrs[s], np.zeros(P, np.uint8), coeff_offset=s * P * channels * 128, out_offset=s * channels * stride,
                                  out_stride=stride) for s in range(S)]
            pcm = fill_guard(np.empty(S * channels * stride, np.float32 if f32 else np.int16))
            if env:
                os.environ.update(env)
            l0 = ctx.launch_count
            k = "k_short" if name == "short" else "k_chain"
            with expect_kernels(ctx, ran={k: 1}, not_ran=ALL_KERNELS - {k}):
                try:
                    if memory == cabi.MEM_DEVICE:
                        d_in, d_out = ctx.device_alloc(spec.nbytes), ctx.device_alloc(pcm.nbytes)
                        ctx.h2d(d_in, spec)
                        ctx.h2d(d_out, pcm)
                        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, d_in, d_out, fmt)
                        ctx.synchronize()
                        ctx.d2h(pcm, d_out)
                        ctx.device_free(d_in)
                        ctx.device_free(d_out)
                    else:
                        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, memory, spec, pcm, fmt)
                finally:
                    if env:
                        for k in env:
                            del os.environ[k]
            assert ctx.launch_count - l0 == 1, (name, ctx.launch_count - l0)       # one k_short (or one k_chain) launch
            outs[(name, batch)] = pcm
            for s in range(S):
                assert chains[s].status == 0 and chains[s].n_samples == n, (name, batch, s, chains[s].n_samples, n)
                got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, :n]
                w = want[s % D]
                if f32:
                    assert bits_equal(got, w), (name, batch, s, mismatch_report(got, w))
                else:
                    assert np.array_equal(got, oracle.quantise_i16(w)), (name, batch, s)
            assert_contained(pcm, write_set(chains, lambda i: channels, fmt), (name, batch))
            for s in range(min(S, 2 * D)):
                assert bits_equal(pwrs[s].data(), refs[s % D].pwr.data()), (name, batch, s)
        for p_ in pwrs:
            p_.close()
    for batch in range(3):
        assert np.array_equal(outs[("short", batch)].view(np.uint8), outs[("chain", batch)].view(np.uint8)), batch
