"""Edge inputs through every kernel that can decode a batch, against the oracle: f32 PCM bit for bit, i16 PCM exactly,
and the final stream state bit for bit.  Each case names the kernel that must have produced its output
(expect_kernels) and checks that its input really reached the edge it is named for.

- Spectrum entry: denormal inputs and outputs, +-0 spectra, +-inf and NaN in single bins, a near-FLT_MAX spectrum that
  overflows inside the IMDCT, blocks loud enough to saturate i16 on both sides, a special value in the packet before a
  long / short boundary (a boundary slot of the one-pass schedule) and in a primer packet of a cut run, and a chain that
  starts from an imported state holding inf / NaN.
- Residue entry: every sign class of a coupled (magnitude, angle) pair, through each shape of the front stages
  (stereo in registers, in both orientations; the shared column of 3-8 channels; the chain kernel's own front half;
  k_prologue for more than 8 channels); an unused floor over a residue holding inf; dense floors holding inf / NaN /
  denormals.
- Floor 1: x lists of rangebits 13-15 whose flagged segments run longer than 4096 bins (the post-shift form of the
  closed-form segment evaluation), 65 posts, every multiplier with posts at range - 1 and above it, and y values up to
  2^24 - 1 that make render_point's product wrap in u32 (audio.rs:354-367, :391-435)."""
import numpy as np
import pytest

import floor1_cases as fc
import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import (ALL_KERNELS, FRONT, RefStream, bits_equal, expect_kernels, launches_are_attributed,
                     make_setup, mismatch_report, mode_sequence)

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

FLT_MAX = np.float32(3.4028235e38)
TINY = np.float32(1.17549435e-38)            # smallest normal f32


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _decode(ctx, chains, entry, coeffs, fmt, total, kw):
    pcm = np.zeros(max(total, 4), np.float32 if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED) else np.int16)
    L.decode_chains(ctx, chains, entry, cabi.MEM_HOST, coeffs, pcm, fmt, **kw)
    return pcm


def _chain_out(pcm, c, C, n, fmt):
    if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR):
        return np.stack([pcm[c.out_offset + k * c.out_stride:c.out_offset + k * c.out_stride + n] for k in range(C)])
    return pcm[c.out_offset:c.out_offset + n * C].reshape(n, C).T


def _check(oracle, pcm, chains, C, wants, pwrs, refs, fmt, what):
    for s, c in enumerate(chains):
        n = wants[s].shape[1]
        assert c.status == 0 and c.n_samples == n, (what, s, c.status, c.n_samples, n)
        got = _chain_out(pcm, c, C, n, fmt)
        if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED):
            assert bits_equal(got, wants[s]), (what, s, mismatch_report(got, wants[s]))
        else:
            assert np.array_equal(got, oracle.quantise_i16(wants[s])), (what, s)
        a, b = pwrs[s].data(), refs[s].pwr.data()
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, s, "state")


def _layout(pwrs, seqs, sizes, C, fmt, n_out, packet_index=None):
    """Chains one after the other in both arenas; planar strides rounded up to multiples of 4."""
    chains, coff, ooff = [], 0, 0
    for s, (mode_ids, prev, nxt) in enumerate(seqs):
        stride = (n_out[s] + 3) & ~3
        chains.append(L.ChainSpec(pwrs[s], mode_ids, prev, nxt, coeff_offset=coff, out_offset=ooff, out_stride=stride,
                                  packet_index=0 if packet_index is None else packet_index[s]))
        coff += sizes[s]
        ooff += stride * C
    return chains, ooff


# ------------------------------------------------------------------------------------------------
# spectrum entry
# ------------------------------------------------------------------------------------------------
SPECTRUM_SHAPES = {   # name: channels, blocksize_0, blocksize_1, share of short blocks, f32 format, kernels that decode it
    "long": (2, 8, 11, 0.0, cabi.OUT_F32_PLANAR, {"k_long"}),
    "short": (2, 8, 8, 0.0, cabi.OUT_F32_PLANAR, {"k_short"}),
    "mid1024": (2, 10, 10, 0.0, cabi.OUT_F32_PLANAR, {"k_mid"}),
    "mid512": (1, 9, 9, 0.0, cabi.OUT_F32_PLANAR, {"k_mid"}),
    "mixed": (2, 8, 11, 0.3, cabi.OUT_F32_PLANAR, {"k_long_s", "k_short_g"}),
    "interleaved": (2, 8, 11, 0.3, cabi.OUT_F32_INTERLEAVED, {"k_chain"}),
    "wide": (10, 8, 11, 0.3, cabi.OUT_F32_PLANAR, {"k_imdct", "k_overlap", "k_save_state"}),
}


def _edge_spectra(rng, C, bf, bs0, bs1, s):
    """Packet spectra of stream s (its edge: see the module docstring); returns [P] arrays [C][n/2]."""
    P = len(bf)
    specs = [(rng.standard_normal((C, (1 << (bs1 if b else bs0)) // 2)) * 0.3).astype(np.float32) for b in bf]
    last = C - 1
    if s == 0:                                   # denormals in and out, +-0
        specs[0][0, :100] = np.float32(1e-42)
        specs[1] *= np.float32(1e-38)
        specs[2] *= np.float32(1e-41)
        specs[3][:] = 0.0
        specs[4][:] = -0.0
        specs[5][last] = -0.0
    elif s == 1:
        # single bins.  Long shape: try_long cuts each of these 24-packet chains into runs of at least 8 packets (its
        # min_run; six stereo chains are far fewer runs than the machine wants), so runs start at packets 8 and 16 and
        # re-transform packets 7 and 15 as their primers.  The inf in packet 7 goes through a primer while that rule holds.
        specs[7][0, 3] = np.inf
        specs[10][last, 9] = np.nan
        specs[13][0, 1] = -np.inf
    elif s == 2:                                 # overflow to inf inside the IMDCT
        specs[6][:] = FLT_MAX * np.where(rng.random(specs[6].shape) < 0.5, -1, 1).astype(np.float32)
    elif s == 3:                                 # i16 saturation on both sides
        specs[4] *= np.float32(1e6)
        specs[9][last] *= np.float32(3e4)
    elif s == 4:                                 # the packet before a long / short boundary, else the one before the last
        edges = [i for i in range(P - 1) if bf[i] != bf[i + 1]]
        assert edges or all(bf), "test should put a special value before a long / short boundary"
        i = edges[len(edges) // 2] if edges else P - 2
        specs[i][0, 5] = np.nan
        specs[i][last, 2] = np.inf
    return specs


@pytest.mark.parametrize("i16", [False, True])
@pytest.mark.parametrize("shape", list(SPECTRUM_SHAPES))
def test_spectrum_edges(ctx, oracle, shape, i16):
    C, bs0, bs1, p_short, fmt, kernels = SPECTRUM_SHAPES[shape]
    if i16:
        fmt = cabi.OUT_I16_PLANAR if fmt == cabi.OUT_F32_PLANAR else cabi.OUT_I16_INTERLEAVED
    rng = np.random.default_rng(700 + list(SPECTRUM_SHAPES).index(shape))
    S, P = 6, 24
    modes = [(0, 0), (1, 0)] if bs0 != bs1 else [(1, 0)]
    su = make_setup(ctx, C, bs0, bs1, modes=modes)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [RefStream(oracle, C, bs0, bs1, modes) for _ in range(S)]
    seqs, coeffs, sizes, wants = [], [], [], []
    for s in range(S):
        if bs0 != bs1:
            bf, prev, nxt = mode_sequence(rng, P, p_short=p_short)
            mode_ids = bf.astype(np.uint8)
        else:
            bf, prev, nxt, mode_ids = np.ones(P, np.uint8), np.ones(P, np.uint8), np.ones(P, np.uint8), np.zeros(P, np.uint8)
        if s == 5:                               # starts from an imported state holding inf / NaN
            n_prev = 1 << (bs1 if bf[0] else bs0)
            st = (rng.standard_normal((C, n_prev // 2)) * 0.5).astype(np.float32)
            st[0, 7], st[C - 1, 100 % (n_prev // 2)], st[0, 11] = np.inf, np.nan, -np.inf
            pwrs[s].set_data(st)
            refs[s].pwr.set_data(st)
        specs = _edge_spectra(rng, C, bf, bs0, bs1, s)
        parts = []
        for i in range(P):
            rc, o = refs[s].spectrum(int(mode_ids[i]), int(prev[i]), int(nxt[i]), specs[i])
            assert rc == 0
            parts.append(o)
        wants.append(np.concatenate(parts, axis=1))
        coeffs.append(np.concatenate([x.ravel() for x in specs]))
        sizes.append(coeffs[-1].size)
        seqs.append((mode_ids, prev, nxt))
    w = wants
    assert np.any((np.abs(w[0]) > 0) & (np.abs(w[0]) < TINY)), "test should exercise denormal outputs"
    assert np.any(np.isnan(w[1])), "test should exercise NaN outputs"
    assert np.any(np.isinf(w[2])) or np.any(np.isnan(w[2])), "test should overflow inside the IMDCT"
    assert np.any(w[3] > 1.0) and np.any(w[3] < -1.0), "test should saturate i16 on both sides"
    assert np.any(np.isnan(w[4])), "test should carry NaN across a boundary"
    assert not np.all(np.isfinite(w[5])), "test should start from a non-finite state"
    # tight planes: a fresh stream's first packet emits nothing, and k_mid takes such chains too
    chains, total = _layout(pwrs, seqs, sizes, C, fmt, [x.shape[1] for x in wants])
    not_ran = (ALL_KERNELS - kernels - {"k_short", "k_row_copy"}) if shape == "mixed" else ALL_KERNELS - kernels
    with expect_kernels(ctx, ran=kernels, not_ran=not_ran):
        pcm = _decode(ctx, chains, cabi.ENTRY_SPECTRUM, np.concatenate(coeffs), fmt, total, {})
    _check(oracle, pcm, chains, C, wants, pwrs, refs, fmt, shape)


# ------------------------------------------------------------------------------------------------
# residue entry: coupled pairs and floors
# ------------------------------------------------------------------------------------------------
CLASSES = np.array([1.5, -2.25, 0.0, -0.0, np.inf, -np.inf, np.nan, 3e-42], np.float32)   # +x -x +0 -0 +inf -inf NaN denormal
_COUPLING_51 = [(0, 1), (2, 3), (0, 4)]
RESIDUE_SHAPES = {   # name: channels, coupling steps, share of short blocks, output format, kernels that decode it
    "stereo": (2, [(0, 1)], 0.0, cabi.OUT_F32_PLANAR, FRONT | {"k_long"}),
    "stereo_swapped": (2, [(1, 0)], 0.0, cabi.OUT_F32_PLANAR, FRONT | {"k_long"}),
    "column": (6, _COUPLING_51, 0.0, cabi.OUT_F32_PLANAR, FRONT | {"k_long"}),
    "chain": (3, [(0, 2), (1, 0)], 0.3, cabi.OUT_F32_INTERLEAVED, {"k_chain"}),
    "wide": (10, [(0, 9), (4, 5), (9, 4)], 0.0, cabi.OUT_F32_PLANAR, {"k_prologue", "k_long"}),
}


@pytest.mark.parametrize("i16", [False, True])
@pytest.mark.parametrize("shape", list(RESIDUE_SHAPES))
def test_residue_edges(ctx, oracle, shape, i16):
    C, coupling, p_short, fmt, kernels = RESIDUE_SHAPES[shape]
    if i16:
        fmt = cabi.OUT_I16_PLANAR if fmt == cabi.OUT_F32_PLANAR else cabi.OUT_I16_INTERLEAVED
    rng = np.random.default_rng(800 + list(RESIDUE_SHAPES).index(shape))
    bs0, bs1, S, P = 8, 11, 4, 22
    floors = [(1, [0, 256, 64, 128, 16, 200]), (3, [0, 128, 40, 90])]
    mappings = [{"coupling": coupling, "floor_of_channel": [c % 2 for c in range(C)]}]
    modes = [(0, 0), (1, 0)]
    su = make_setup(ctx, C, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [RefStream(oracle, C, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    pairs = [(m, a) for m in CLASSES for a in CLASSES]      # every (magnitude, angle) class pair
    seqs, coeffs, dense, kinds, ys, sizes, wants = [], [], [], [], [], [], []
    n_pairs = 0
    hit = {"unused_inf": False, "dense_special": False}
    for s in range(S):
        bf, prev, nxt = mode_sequence(rng, P, p_short=p_short)
        mode_ids = bf.astype(np.uint8)
        parts = []
        for i in range(P):
            n2 = (1 << (bs1 if bf[i] else bs0)) // 2
            res = (rng.standard_normal((C, n2)) * 0.5).astype(np.float32)
            fl = []
            for c in range(C):
                mult, xs = floors[c % 2]
                fl.append([int(v) for v in rng.integers(0, [256, 128, 86, 64][mult - 1], len(xs))])
            if (s * P + i) % 4 == 3:
                # floor edges, in packets of their own (their NaN would hide how a pair was decoupled)
                c0, c1 = (s + i) % C, (s + i + 1) % C
                res[c0, 1 + i] = np.inf                  # unused floor over a residue holding inf: 0 x inf = NaN
                fl[c0] = None
                d = (rng.random(n2) + 0.1).astype(np.float32)
                d[2], d[5], d[8], d[11] = np.inf, np.nan, np.float32(1e-40), -0.0
                fl[c1] = d                                # dense floor holding inf / NaN / denormals
                hit["unused_inf"] = hit["dense_special"] = True
            else:
                # one class pair per packet, in one bin of one coupling step: a NaN or inf there reaches only the
                # channels the reference's decoupling sends it to (audio.rs:762-777)
                m, a = coupling[n_pairs % len(coupling)]
                res[m, 7], res[a, 7] = pairs[n_pairs % len(pairs)]
                n_pairs += 1
            rc, o = refs[s].packet(int(mode_ids[i]), int(prev[i]), int(nxt[i]), res, fl)
            assert rc == 0
            parts.append(o)
            k_, y_, d_ = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
            kinds.append(k_)
            ys.append(y_)
            dense.append((d_ if d_ is not None else np.zeros_like(res)).ravel())
            coeffs.append(res.ravel())
        wants.append(np.concatenate(parts, axis=1))
        sizes.append(sum(C * ((1 << (bs1 if b else bs0)) // 2) for b in bf))
        seqs.append((mode_ids, prev, nxt))
    assert all(hit.values()) and n_pairs >= len(pairs), (hit, n_pairs)
    assert any(np.any(np.isnan(w)) for w in wants), "test should carry NaN to the output"
    chains, total = _layout(pwrs, seqs, sizes, C, fmt, [x.shape[1] for x in wants], packet_index=[s * P for s in range(S)])
    kw = dict(floor_kind=np.concatenate(kinds), floor1_y=np.concatenate(ys), dense_floor=np.concatenate(dense))
    with expect_kernels(ctx, ran=kernels, not_ran=ALL_KERNELS - kernels):
        pcm = _decode(ctx, chains, cabi.ENTRY_RESIDUE, np.concatenate(coeffs), fmt, total, kw)
    _check(oracle, pcm, chains, C, wants, pwrs, refs, fmt, shape)


# ------------------------------------------------------------------------------------------------
# floor 1: long segments, 65 posts, every multiplier, the clamp, wrapping render_point
# ------------------------------------------------------------------------------------------------
def _long_segment_xs(rng, rangebits, n2):
    """65 posts: [0, 2^rangebits], 40 posts below n/2 and 23 more than 4096 bins above n/2.  Returns the list and the
    bins between the last post below n/2 and the first one at or above it (every flagged segment that covers bin n/2 - 1
    spans at least that many)."""
    lo = rng.choice(np.arange(1, n2 - 1), 40, replace=False)
    hi = rng.choice(np.arange(n2 + 4200, 1 << rangebits), 23, replace=False)
    xs = [0, 1 << rangebits] + [int(v) for v in rng.permutation(np.concatenate([lo, hi]))]
    below = max(x for x in xs if x < n2)
    above = min(x for x in xs if x >= n2)
    return xs, above - below


def _wild_y(rng, mult, nposts):
    rng_y = [256, 128, 86, 64][mult - 1]
    y = [int(rng.integers(rng_y - 1, 256)), int(rng.integers(0, 256))]      # posts 0 / 1: at range - 1 and above
    for _ in range(nposts - 2):
        r = rng.random()
        y.append(0 if r < 0.3 else int(rng.integers(1, 40)) if r < 0.6 else int(rng.integers(rng_y - 1, 2 * rng_y))
                 if r < 0.8 else int(rng.integers(1 << 20, 1 << 24)))
    return y


@pytest.mark.parametrize("rangebits", [13, 14, 15])
@pytest.mark.parametrize("n", [2048, 1024, 512])
def test_floor1_long_segments_and_wild_posts(ctx, oracle, n, rangebits):
    rng = np.random.default_rng(900 + n + rangebits)
    bs = n.bit_length() - 1
    bs0, bs1 = (8, 11) if n == 2048 else (bs, bs)
    n2 = n // 2
    C, S, P = 2, 5, 6
    floors = []
    for mult in (1, 2, 3, 4):
        xs, span = _long_segment_xs(rng, rangebits, n2)
        assert len(xs) == 65 and span > 4096 and max(x for x in xs if x < n2) < n2, "test should need the post-shift"
        floors.append((mult, xs))
    mappings = [{"coupling": [(0, 1)], "floor_of_channel": [0, 1]}, {"coupling": [(1, 0)], "floor_of_channel": [2, 3]}]
    modes = [(1, 0), (1, 1)]
    su = make_setup(ctx, C, bs0, bs1, modes=modes, mappings=mappings, floors=floors)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    refs = [RefStream(oracle, C, bs0, bs1, modes, mappings, floors) for _ in range(S)]
    seqs, coeffs, kinds, ys, sizes, wants = [], [], [], [], [], []
    wraps = at_edge = above = 0
    for s in range(S):
        mode_ids = rng.integers(0, 2, P).astype(np.uint8)
        parts = []
        for i in range(P):
            res = (rng.standard_normal((C, n2)) * 0.5).astype(np.float32)
            fl = []
            for c in range(C):
                mult = floors[mappings[mode_ids[i]]["floor_of_channel"][c]][0]
                y = _wild_y(rng, mult, 65)
                prods, fy, _ = fc.unwrap(floors[mappings[mode_ids[i]]["floor_of_channel"][c]][1], mult, y)
                wraps += sum(v >= 1 << 32 for v in prods)
                at_edge += sum(v == [256, 128, 86, 64][mult - 1] - 1 for v in fy)
                above += sum(v > [256, 128, 86, 64][mult - 1] - 1 for v in fy)
                fl.append(y)
            rc, o = refs[s].packet(int(mode_ids[i]), 1, 1, res, fl)
            assert rc == 0
            parts.append(o)
            k_, y_, _ = L.DecodedPacket(int(mode_ids[i]), res, fl).pack()
            kinds.append(k_)
            ys.append(y_)
            coeffs.append(res.ravel())
        wants.append(np.concatenate(parts, axis=1))
        sizes.append(P * C * n2)
        seqs.append((mode_ids, np.ones(P, np.uint8), np.ones(P, np.uint8)))
    assert wraps and at_edge and above, ("test should wrap render_point and put posts at range - 1 and above", wraps, at_edge, above)
    kernels = FRONT | {"k_long" if n == 2048 else "k_mid"}
    for fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR):        # each from empty streams; refs hold the end states
        for p_ in pwrs:
            p_.reset()
        chains, total = _layout(pwrs, seqs, sizes, C, fmt, [x.shape[1] for x in wants], packet_index=[s * P for s in range(S)])
        with expect_kernels(ctx, ran=kernels, not_ran=ALL_KERNELS - kernels):
            pcm = _decode(ctx, chains, cabi.ENTRY_RESIDUE, np.concatenate(coeffs), fmt, total,
                          dict(floor_kind=np.concatenate(kinds), floor1_y=np.concatenate(ys)))
        _check(oracle, pcm, chains, C, wants, pwrs, refs, fmt, (n, rangebits, fmt))
