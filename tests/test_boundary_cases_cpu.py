"""The boundary-site table and plan model (boundary_cases.py) without a GPU: the cases reach every site at the SM
counts of H100 parts, the runtime-ls sites at every blocksize_0 the long-block kernel takes, the model's walk agrees
with the oracle's overlap rules, and the oracle decodes every routing row."""
import numpy as np
import pytest

import boundary_cases as bc
from helpers import RefStream

SM_COUNTS = (132, 114)      # H100 SXM5 / PCIe


@pytest.mark.parametrize("sm", SM_COUNTS)
def test_rows_reach_every_site(sm):
    """Each row reaches the sites it is listed for, and together they reach every site of the table: a site no row
    reaches is a boundary body no GPU test decodes."""
    reached = set()
    for row in bc.ROWS:
        got = bc.case_sites(bc.CASES[row.case], sm, row.env)
        assert row.sites <= got, (row.case, row.env, sorted(row.sites - got))
        reached |= got
    assert reached == set(bc.SITES), sorted(set(bc.SITES) - reached)


@pytest.mark.parametrize("sm", SM_COUNTS)
def test_host_chunks_reach_the_same_sites(sm):
    """A host-memory batch in three chunks plans each chunk's rounds and cuts on its own; the rows still reach the sites
    they are listed for (the GPU rows run every case that way too)."""
    for row in bc.ROWS:
        got = bc.case_sites(bc.CASES[row.case], sm, dict(row.env or {}, **bc.CHUNKS), "host")
        missing = row.sites - got - {"R6"}       # (a chunk may hold no chain outside the pass)
        assert not missing, (row.case, row.env, sorted(missing))


@pytest.mark.parametrize("bs0", bc.RUNTIME_LS_BS0)
def test_runtime_ls_sites_at_every_blocksize_0(bs0):
    """k_long's first_short and last_short bodies with ls at run time, at ls = (2048 - 2^bs0) / 4 for blocksize_0 6-10:
    the runtime-ls case of that blocksize reaches them on k_long, and only there."""
    c = bc.CASES[f"runtime_ls_{bs0}"]
    env = bc.ROUNDS if bs0 == 8 else None
    ps = bc.plans(c, 132, env)
    assert {f"T{bs0}F", f"T{bs0}E"} <= set().union(*(p.sites for p in ps))
    assert all(p.launches["k_long_s"] == 0 for p in ps)
    lr = [x for p in ps for x in p.long if x.first_short or x.last_short]
    assert lr and all(x.kernel == "k_long" and x.ls == (2048 - (1 << bs0)) // 4 for x in lr)
    if bs0 != 8:        # (at 8 the pass takes the same case: k_long_s at its compile-time LS)
        assert bc.case_sites(c, 132) >= {f"T{bs0}F", f"T{bs0}E"}
    else:
        assert not bc.case_sites(c, 132) & {"T8F", "T8E"}


@pytest.mark.parametrize("bs0", [6, 7, 8, 9, 10, 11])
def test_walk_agrees_with_the_oracle_overlap_rules(oracle, bs0):
    """The model's walk_chain stops where the oracle does: a slope shorter than the state stops with BAD_FORMAT and
    empties it (audio.rs:1107-1111), ls + plen > n stops with MISMATCH (where the reference would index out of range).
    Every (block, flags) on every state length a stream of this setup or an imported one can hold."""
    C = 1
    rng = np.random.default_rng(bs0)
    plens = sorted({0, 16, 32, 64, 128, 256, 512, 1024} | {(1 << bs0) // 2})
    for plen in plens:
        for bf in (0, 1):
            for pf in (0, 1):
                for nf in (0, 1):
                    ref = RefStream(oracle, C, bs0, 11, [(0, 0), (1, 0)])
                    if plen:
                        ref.pwr.set_data(rng.standard_normal((C, plen)).astype(np.float32))
                    n2 = (1 << (11 if bf else bs0)) // 2
                    rc, _ = ref.spectrum(bf, pf, nf, rng.standard_normal((C, n2)).astype(np.float32))
                    w = bc.walk(bs0, 11, (plen > 0, plen), [bf], [pf], [nf])
                    assert w.status == rc, (bs0, plen, bf, pf, nf, w.status, rc)
                    if rc == bc.BAD_FORMAT:
                        assert w.end == (False, 0) and ref.pwr.is_empty()
                    if rc == bc.OK:
                        g = w.packets[0][1]
                        assert w.end == (True, g.re - g.rs) == (True, len(ref.pwr))


def test_routing_follows_the_walk_rules():
    """The routing rows: a long block with prev flag 0 on a 1024-sample state stops (its slope is shorter), a short
    block on one too; a long block with prev flag 0 after one with next flag 0 makes two long segments; one with prev
    flag 1 on a 128-sample state goes to the chain kernel."""
    w = bc.walk(8, 11, (True, 1024), [1], [0], [1])
    assert w.status == bc.BAD_FORMAT and not w.packets
    w = bc.walk(8, 11, (True, 1024), [0], [1], [1])
    assert w.status == bc.BAD_FORMAT and not w.packets
    (bf, pf, nf), = bc.stream("L S L L10 L01 L")
    segs = bc.segment(8, bc.walk(8, 11, (False, 0), bf, pf, nf))
    assert [(s.kind, s.n, s.first_short, s.last_short) for s in segs] == [
        ("long", 1, False, True), ("short", 1, False, False), ("long", 2, True, True), ("long", 2, True, False)]
    (bf, pf, nf), = bc.stream("L S L11 L")
    segs = bc.segment(8, bc.walk(8, 11, (False, 0), bf, pf, nf))
    assert [(s.kind, s.n) for s in segs] == [("long", 1), ("short", 1), ("chain", 1), ("long", 1)]


@pytest.mark.parametrize("name", sorted(bc.CASES))
def test_oracle_decodes_every_case(oracle, name):
    """Every packet of every case decodes in the oracle with rc 0 (the routing rows' inconsistent flags included), and
    the model's sample counts and end states are the oracle's."""
    c = bc.CASES[name]
    rng = np.random.default_rng(1)
    for s, st in enumerate(c.streams):
        ref = RefStream(oracle, 1, c.bs0, 11, [(0, 0), (1, 0)])
        state = (False, 0)
        for b, (bf, pf, nf) in enumerate(st):
            n = 0
            for i in range(len(bf)):
                n2 = (1 << (11 if bf[i] else c.bs0)) // 2
                rc, pcm = ref.spectrum(int(bf[i]), int(pf[i]), int(nf[i]), rng.standard_normal((1, n2)).astype(np.float32))
                assert rc == 0, (name, s, b, i)
                n += pcm.shape[1]
            w = bc.walk(c.bs0, 11, state, bf, pf, nf)
            assert (w.status, w.samples, w.end) == (0, n, (True, len(ref.pwr))), (name, s, b)
            state = w.end
