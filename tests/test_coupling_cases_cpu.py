"""The inverse-coupling cases of coupling_cases.py without a GPU: the numpy restatement against the oracle, the cases'
reach over sites and topology classes, and the inputs every case feeds each coupling step."""
import numpy as np
import pytest

import coupling_cases as cc

ALL_CASES = cc.cases() + cc.vq_cases() + cc.tap_cases()


def test_classes_match_the_kernel_edges_module():
    import test_kernel_edges
    assert np.array_equal(cc.CLASSES.view(np.uint32), test_kernel_edges.CLASSES.view(np.uint32))


def test_every_site_reaches_every_class_it_can_take():
    got = cc.reached(ALL_CASES)
    missing = {s: sorted(want - got.get(s, set())) for s, want in cc.SITE_CLASSES.items()}
    assert not any(missing.values()), missing
    for c in ALL_CASES:
        assert c.site in cc.SITES, c
        assert c.classes() <= cc.SITE_CLASSES[c.site], (c, sorted(c.classes() - cc.SITE_CLASSES[c.site]))
    assert {c.C for c in cc.tap_cases()} == set(range(1, 13))


def test_inverse_couple_matches_the_oracle_on_every_class_pair(oracle):
    m = np.repeat(cc.CLASSES, 8)
    a = np.tile(cc.CLASSES, 8)
    for mm, aa in ((m, a), (-m, a), (m * np.float32(1e-38), a * np.float32(3))):     # and denormal sums, rounding
        gm, ga = oracle.inverse_couple(mm, aa)
        wm, wa = cc.inverse_couple(mm, aa)
        assert np.all(cc.same_bits(wm, gm)) and np.all(cc.same_bits(wa, ga))


@pytest.mark.parametrize("case", ALL_CASES, ids=repr)
def test_step_loop_matches_the_oracle_and_is_order_sensitive(oracle, case):
    """Per mapping: the restatement's decoupling of the case's probe columns and random bins equals the oracle's step
    loop (lwo_inverse_couple in reverse), and, with >= 2 steps, differs in bits from the steps run forward (unless the
    list reads the same both ways) and from magnitude and angle exchanged -- else the case could not tell those
    mistakes apart."""
    rng = np.random.default_rng(5)
    for mp in case.mappings:
        fin, nf = cc.mapping_pool(case.C, mp)
        res = np.concatenate([fin, nf, (rng.standard_normal((case.C, 64)) * 0.5).astype(np.float32)], axis=1)
        want = res.copy()
        for m, a in reversed(mp):
            want[m], want[a] = oracle.inverse_couple(want[m], want[a])
        got = cc.decouple(res, mp)
        assert np.all(cc.same_bits(got, want)), (case, mp)
        if len(mp) >= 2:
            if mp != mp[::-1]:                # (a palindrome is the same list either way: see the next test)
                assert cc.differ_in_bits(cc.decouple(res, mp, forward=True), got), (case, mp, "forward order gives the same bits")
            assert cc.differ_in_bits(cc.decouple(res, mp, exchange=True), got), (case, mp, "exchanged roles give the same bits")


@pytest.mark.parametrize("case", ALL_CASES, ids=repr)
def test_probe_columns_feed_each_step_its_classes(case):
    """Every step that no later step shares a channel with has a column for each of the 64 class pairs, every other step
    for the pairs a decoupling can hand it (at least 8, one of them two finite nonzero values).  A case's packets carry
    every finite pair of every step whose column stays finite in every channel, and every step a non-finite pair."""
    for mp in case.mappings:
        probes = cc.probe_columns(case.C, mp)
        free = set(cc.free_steps(mp))
        fin, nf = cc.mapping_pool(case.C, mp)
        cols = np.concatenate([fin, nf], axis=1)
        seen = cc.step_classes(cols, mp) if mp else {}
        for s in range(len(mp)):
            for p in {p for p in probes[s] if cc.finite_pair(p)} - seen[s]:     # only a column with inf / NaN elsewhere
                col = probes[s][p][:, None]
                assert not (np.isfinite(col).all() and np.isfinite(cc.decouple(col, mp)).all()), (case, s, p)
            if s in free:
                assert len(probes[s]) == 64, (case, mp[s], sorted(set(cc.PAIRS) - set(probes[s])))
            assert len(seen[s]) >= 8 and seen[s] & {(0, 0), (0, 1), (1, 0), (1, 1)}, (case, s, sorted(seen[s]))
            assert any(not cc.finite_pair(p) for p in seen[s]), (case, s)


def test_synth_packet_equals_the_restatement_then_synth_spectrum(oracle):
    """The oracle's whole residue stage (synth_packet: coupling, floor x residue, IMDCT, overlap) equals the restatement's
    decoupling times the floor, through synth_spectrum, on every case's mappings."""
    rng = np.random.default_rng(6)
    for case in ALL_CASES:
        for mp in case.mappings[:4] + case.mappings[-1:]:
            n2 = 128
            fin, _ = cc.mapping_pool(case.C, mp)
            res = (rng.standard_normal((case.C, n2)) * 0.5).astype(np.float32)
            k = min(n2 - 8, fin.shape[1])
            res[:, 4:4 + k] = fin[:, :k]
            dense = [(rng.random(n2) + 0.1).astype(np.float32) for _ in range(case.C)]
            a, b = oracle.Pwr(case.C, 8), oracle.Pwr(case.C, 8)
            rc1, got = oracle.synth_packet(8, 8, 0, 1, 1, mp, dense, res, a)
            spec = cc.decouple(res, mp) * np.stack(dense)
            rc2, want = oracle.synth_spectrum(8, 8, 0, 1, 1, spec, b)
            assert rc1 == rc2 == 0
            assert np.all(cc.same_bits(a.data(), b.data())), (case, mp)


def test_handover_modes_differ_between_consecutive_packets_of_a_cta():
    for grid, n_pk in ((1056, 2400), (528, 1200), (7, 40)):
        modes = cc.handover_modes(n_pk, grid, 14)
        a, b = modes[:-grid], modes[grid:]
        assert np.all(a % 2 != b % 2) and np.all(a // 2 != b // 2)


@pytest.mark.parametrize("case", ALL_CASES, ids=repr)
def test_every_case_with_several_steps_tells_the_orders_apart(case):
    """A list that reads the same both ways cannot tell steps run forward from steps run in reverse; every case with a
    multi-step list keeps one that does not, so that a kernel running its steps forward fails on it."""
    multi = [mp for mp in case.mappings if len(mp) >= 2]
    assert not multi or any(mp != mp[::-1] for mp in multi), (case, multi)


@pytest.mark.parametrize("case", cc.cases(), ids=repr)
def test_finite_probes_reach_the_pcm(case):
    """The chains of finite probes (finite_chain) carry every finite probe column of each mapping, every bin of theirs
    stays finite through the decoupling, and their floors are never unused -- so the PCM shows every probe.  Each
    packet of the non-finite chains carries exactly one non-finite column."""
    rng = np.random.default_rng(8)
    n0, n1 = (1 << case.bs0) // 2, (1 << case.bs1) // 2
    assert all(cc.floor_kind(j, c, unused=False) != cc.FLOOR_UNUSED for j in range(12) for c in range(case.C))
    for mp in case.mappings:
        fin, nf = cc.mapping_pool(case.C, mp)
        chain = cc.finite_chain(rng, case.C, fin, n0, n1)
        carried = np.concatenate([res[:, 4:res.shape[1] - 4] for _, res in chain], axis=1)
        assert carried.shape[1] >= fin.shape[1] and np.array_equal(carried[:, :fin.shape[1]].view(np.uint32), fin.view(np.uint32))
        for bf, res in chain:
            assert res.shape == (case.C, n1 if bf else n0)
            assert np.isfinite(cc.decouple(res, mp)).all(), (case, mp)
        for bf, res in cc.nonfinite_chain(rng, case.C, nf, n0, n1):
            bad = ~np.isfinite(res).all(axis=0)
            assert bad.sum() == 1 and bad[1], (case, mp)


def test_packer_takes_fixed_couplings():
    import vorbis_packer as vp
    couplings = [[], [(0, 1)], [(1, 0), (0, 1), (1, 0)]]
    spec = vp.StreamSpec(np.random.default_rng(1), channels=2, couplings=couplings)
    assert [m["coupling"] for m in spec.mappings] == couplings
    assert spec.modes == [(0, 0), (1, 0), (0, 1), (1, 1), (0, 2), (1, 2)]
