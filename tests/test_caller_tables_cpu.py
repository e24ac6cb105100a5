"""The oracle decodes with a caller's own blocksize tables (oracle.Tables.from_arrays), and the table sets of
caller_tables are what they claim to be: the GPU tests hold every kernel to the oracle fed the same tables."""
import numpy as np
import pytest

import caller_tables as ct
from helpers import RefStream, bits_equal

MODES = [(0, 0), (1, 0)]
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
PAIRS = [(6, 6), (6, 7), (7, 8), (8, 9), (9, 10), (10, 11), (11, 12), (12, 13), (13, 13)]   # every blocksize, both slots


def stream_pcm(oracle, bs0, bs1, tables, residue, seed=0):
    """PCM and end state of a short block sequence (short, long after short, long, short after long) through the oracle."""
    rng = np.random.default_rng(seed)
    ref = RefStream(oracle, 2, bs0, bs1, MODES, floors=[FLOOR], tables=tables)
    seq = [(1, 1, 0), (0, 1, 1), (1, 0, 1), (1, 1, 1), (1, 1, 0), (0, 1, 1), (0, 1, 1), (1, 0, 1)]
    out = []
    for bf, pf, nf in seq:
        n2 = (1 << (bs1 if bf else bs0)) // 2
        x = (rng.standard_normal((2, n2)) * 0.25).astype(np.float32)
        if residue:
            y = [[int(v) for v in rng.integers(0, 128, len(FLOOR[1]))] for _ in range(2)]
            rc, o = ref.packet(bf, pf, nf, x, y)
        else:
            rc, o = ref.spectrum(bf, pf, nf, x)
        assert rc == 0
        out.append(o)
    return np.concatenate(out, axis=1), ref.pwr.data()


@pytest.mark.parametrize("bs0,bs1", PAIRS)
def test_canonical_arrays_decode_like_the_generated_tables(oracle, bs0, bs1):
    tabs = ct.oracle_pair(oracle, ct.table_set("canonical", bs0, bs1))
    for residue in (False, True):
        got, got_end = stream_pcm(oracle, bs0, bs1, tabs, residue)
        want, want_end = stream_pcm(oracle, bs0, bs1, None, residue)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (bs0, bs1, residue)
        assert np.array_equal(got_end.view(np.uint32), want_end.view(np.uint32)), (bs0, bs1, residue)
    x = np.random.default_rng(bs1).standard_normal(1 << (bs1 - 1)).astype(np.float32)
    assert np.array_equal(oracle.inverse_mdct(x, bs1, tables=tabs[1]).view(np.uint32), oracle.inverse_mdct(x, bs1).view(np.uint32))


@pytest.mark.parametrize("bs0,bs1", [(8, 11), (10, 10), (6, 13)])
def test_other_tables_change_the_output(oracle, bs0, bs1):
    """f64 and scrambled tables give other PCM than the generated ones; split tables too, and each half of a split pair
    on the packets that read it -- short packets (tab[0]) and long ones (tab[1])."""
    want, _ = stream_pcm(oracle, bs0, bs1, None, False)
    for name in ("f64", "scrambled", "split_bs0", "split_bs1"):
        got, _ = stream_pcm(oracle, bs0, bs1, ct.oracle_pair(oracle, ct.table_set(name, bs0, bs1)), False)
        assert not bits_equal(got, want), name
    # a long block on long neighbours reads tab[1] only, a short block on short neighbours tab[0] only
    for bf, name, other in ((1, "split_bs1", "split_bs0"), (0, "split_bs0", "split_bs1")):
        n2 = (1 << (bs1 if bf else bs0)) // 2
        x = np.random.default_rng(bf).standard_normal((1, n2)).astype(np.float32)
        pcm = {}
        for nm in (None, name, other):
            p = oracle.Pwr(1, bs1)
            tabs = None if nm is None else ct.oracle_pair(oracle, ct.table_set(nm, bs0, bs1))
            for _ in range(2):
                rc, o = oracle.synth_spectrum(bs0, bs1, bf, bf, bf, x, p, tables=tabs)
                assert rc == 0
            pcm[nm] = o
        assert not bits_equal(pcm[name], pcm[None]), (bf, name)
        if bs0 != bs1 or bf:
            assert bits_equal(pcm[other], pcm[None]), (bf, other)


def test_tables_of_another_blocksize_are_refused(oracle):
    t = ct.canonical(8)
    with pytest.raises(ValueError):
        oracle.Tables.from_arrays(9, t["a"], t["b"], t["c"], t["window"], t["bitrev"])
    with pytest.raises(ValueError):
        oracle.synth_spectrum(8, 9, 1, 1, 1, np.zeros((1, 256), np.float32), oracle.Pwr(1, 9),
                              tables=ct.oracle_pair(oracle, [t, t]))


@pytest.mark.parametrize("bs", range(6, 14))
def test_f64_tables_differ_where_a_float64_libm_rounds_otherwise(bs):
    assert ct.differing(ct.f64_raw(bs), ct.canonical(bs)) == ct.F64_DIFFERS[bs]
    assert all(ct.differing(ct.f64(bs), ct.canonical(bs)))
    f, g = ct.f64(bs), ct.canonical(bs)
    for k in ct.ARRAYS:                           # rounding, not a different formula: a few f32 epsilons at most
        assert np.max(np.abs(f[k].astype(np.float64) - g[k])) <= 2 * float(np.finfo(np.float32).eps), k
    assert np.array_equal(f["bitrev"], g["bitrev"])


@pytest.mark.parametrize("bs", range(6, 14))
def test_scrambled_tables_hold_the_values_a_kernel_could_get_away_with(bs):
    t, g = ct.scrambled(bs), ct.canonical(bs)
    assert np.array_equal(t["bitrev"], g["bitrev"])
    for k in ct.ARRAYS:
        v = t[k]
        assert v.dtype == np.float32 and v.shape == g[k].shape, k
        bits = v.view(np.uint32)
        assert np.any(bits == 0) and np.any(bits == 0x80000000), (k, "+0 and -0")
        assert np.any(v == 1.0) and np.any(v == -1.0), (k, "+-1.0")
        sub = (v != 0) & (np.abs(v) < np.finfo(np.float32).tiny)
        assert np.count_nonzero(sub) == 3, k
        assert np.all(np.abs(v) <= 1.0) and np.all(np.isfinite(v))
        assert np.count_nonzero(bits == g[k].view(np.uint32)) < max(3, v.size // 50), k
    assert all(np.array_equal(ct.scrambled(bs)[k], t[k]) for k in ct.ARRAYS)       # one table per blocksize
