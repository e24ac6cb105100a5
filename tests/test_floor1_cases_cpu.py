"""floor1_cases.py on the CPU: every post layout reaches the edge it is named for, the Python-integer walk equals the
oracle's floor-1 curve, the device's floor-1 source run on the host (tests/emu/floor1_emu.cpp) equals the walk on every
layout at every n/2 from 32 to 4096, and prepare_floor1 refuses x lists whose post 0 is not at x = 0."""
import ctypes as C

import numpy as np
import pytest

import floor1_cases as fc
from test_floor1_emu import build

N2S = [32, 64, 128, 256, 512, 1024, 2048, 4096]


def _edge_holds(lay):
    """Whether lay reaches its edge at lay.n2; returns (holds, what was found)."""
    n2, name = lay.n2, lay.name
    prods, fy, flag = fc.unwrap(lay.xs, lay.mult, lay.y)
    posts = fc.flagged_posts(lay.xs, lay.mult, lay.y)
    segs = [s for s in lay.segments() if s[0] < n2]
    px = [x for x, _ in posts]
    if name.startswith("two_posts"):
        tail = lay.xs[1] < n2
        return len(lay.xs) == 2 and len(segs) == (2 if tail else 1) and (tail or lay.xs[1] > n2), segs
    if name == "full_table":
        return len(lay.xs) == 65 and all(flag) and px[-1] < n2 and len(lay.segments()) + 1 == 66, (len(px), px[-1])
    if name.startswith("end_at_n2"):
        d = int(name[len("end_at_n2"):])
        return px[-1] == n2 + d and (d >= 0 or segs[-1][2] - segs[-1][0] == 1), (px[-1], segs[-1])
    if name == "long_x_list":
        over = [s for s in segs if s[0] <= n2 - 1 < s[2]]
        return lay.xs[1] == 1 << 15 and len(over) == 1 and over[0][2] - over[0][0] > 4096, over
    if name.startswith("steep"):
        top = 255 if lay.mult == 1 else 252
        dys = {(s[2] - s[0], s[3] - s[1]) for s in segs}
        base = any(abs(dy) >= adx > 1 for adx, dy in dys)
        return (1, top) in dys and (1, -top) in dys and any(dy == 0 for _, dy in dys) and base, sorted(dys)
    if name == "word_boundaries":
        pset = set(x for x in px if x < n2)
        quads = {}
        for x in pset:
            quads[x >> 2] = quads.get(x >> 2, 0) + 1
        want_quads = {2, 3, 4} if n2 >= 96 else set()
        full = any(all(32 * w + b in pset for b in range(32)) for w in range(n2 // 32))
        bounds = {x for k in range(1, min(n2 // 32, 5)) for x in (32 * k - 1, 32 * k)} | {31}
        return bounds <= pset and want_quads <= set(quads.values()) and full, (sorted(pset)[:40], quads)
    if name.startswith("post64"):
        on = name.endswith("on")
        xs_sorted = sorted(range(len(lay.xs)), key=lambda i: lay.xs[i])
        between = any(not flag[xs_sorted[k]] and flag[xs_sorted[k - 1]] and flag[xs_sorted[k + 1]]
                      for k in range(1, len(xs_sorted) - 1))
        return len(lay.xs) == 65 and flag[64] == on and between, (flag[64], between)
    if name.startswith("clamp"):
        top = fc.RANGE[lay.mult - 1] - 1
        vals = [v for v, f in zip(fy, flag) if f and v < 1 << 31]
        return top in vals and any(v > top for v in vals), sorted(set(vals))[-5:]
    if name == "wrap":
        return any(p >= 1 << 32 for p in prods) and max(lay.y) >= 1 << 20, max(prods)
    raise AssertionError(f"no edge check for {name}")


@pytest.mark.parametrize("n2", N2S)
def test_layouts_reach_their_edges(n2):
    lays = fc.layouts(n2)
    names = {lay.name for lay in lays}
    for f in fc.CONSTRUCTORS:
        if n2 >= 128 or f is not fc.full_table:
            assert f(np.random.default_rng(n2), n2), f"{f.__name__} gives no layout at n/2 = {n2}"
    assert "wrap" in names and {f"clamp_m{m}" for m in (1, 2, 3, 4)} <= names
    for lay in lays:
        ok, found = _edge_holds(lay)
        assert ok, (lay, lay.edge, found)


def test_walk_renders_render_line_by_hand():
    """Two hand-worked floors: a two-post line with a flat tail, and a truncated steep line."""
    # multiplier 2, posts 0 -> 10 (final y 20 -> 40 after the multiplier) over 4 bins, tail at 40 to n/2 = 8
    assert fc.walk([0, 4], 2, [10, 20], 8) == [20, 25, 30, 35, 40, 40, 40, 40]
    # multiplier 1, 255 -> 0 over 10 bins (base -25, 5 / 10 of a step more every bin), truncated at 6 bins
    assert fc.walk([0, 10], 1, [255, 0], 6) == [255, 230, 204, 179, 153, 128]


@pytest.mark.parametrize("n2", N2S)
def test_walk_matches_the_oracle(oracle, n2):
    db = oracle.inverse_db_table()
    for lay in fc.layouts(n2):
        fl = oracle.make_floor1(lay.mult, lay.xs)
        final_y, step2 = oracle.floor1_amplitude(fl, lay.y)
        _, fy, flag = fc.unwrap(lay.xs, lay.mult, lay.y)
        top = fc.RANGE[lay.mult - 1] - 1
        assert final_y.tolist() == [min(v, top) for v in fy] and step2.astype(bool).tolist() == flag, lay
        for m in sorted({n2, 32, 4096}):
            want = lay.walk(m)
            assert len(want) == m and all(0 <= v <= 255 for v in want), lay
            assert oracle.floor1_curve_y(fl, final_y, step2, m).tolist() == want, (lay, m)
            assert np.array_equal(oracle.floor1_synthesis(fl, final_y, step2, m), db[np.array(want)]), (lay, m)


def _emu(L, lay, n2):
    xa, ya = np.array(lay.xs, np.uint32), np.array(lay.y, np.uint32)
    closed, render, packed = np.zeros(n2, np.uint32), np.zeros(n2, np.uint8), np.zeros(n2, np.uint8)
    rc = L.lwb_emu_floor1(lay.mult, xa.ctypes.data_as(C.c_void_p), len(lay.xs), ya.ctypes.data_as(C.c_void_p), n2,
                          closed.ctypes.data_as(C.c_void_p), render.ctypes.data_as(C.c_void_p), packed.ctypes.data_as(C.c_void_p))
    return rc, closed, render, packed


@pytest.mark.parametrize("n2", N2S)
def test_emu_matches_the_walk_at_every_n2(n2):
    """Layouts built for n2, evaluated at every n/2 of N2S: the closed form (d_floor1_y_at), the DDA render
    (d_floor1_render_segment) and the packed segments (d_floor1_pack_segment / d_floor1_seg_y)."""
    L = C.CDLL(build())
    for lay in fc.layouts(n2):
        for m in N2S:
            rc, closed, render, packed = _emu(L, lay, m)
            assert rc == 0, (lay, m, rc)
            want = np.array(lay.walk(m), np.uint32)
            assert np.array_equal(closed, want), (lay, m, np.nonzero(closed != want)[0][:5])
            assert np.array_equal(render.astype(np.uint32), want), (lay, m, np.nonzero(render != want)[0][:5])
            assert np.array_equal(packed.astype(np.uint32), want), (lay, m, np.nonzero(packed != want)[0][:5])


def test_prepare_floor1_refuses_x_lists_not_starting_at_zero():
    """Posts 0 and 1 bracket every other post in these lists, so only post 0 away from x = 0 is wrong with them."""
    L = C.CDLL(build())
    LWB_ERR_BAD_FORMAT = 1
    for xs in ([5, 100, 50], [1, 2], [32767, 32768], [3, 64, 5, 10, 63]):
        lay = fc.Layout.__new__(fc.Layout)
        lay.mult, lay.xs, lay.y = 1, xs, [10] * len(xs)
        rc, *_ = _emu(L, lay, 32)
        assert rc == LWB_ERR_BAD_FORMAT, (xs, rc)
    lay = fc.layouts(32)[0]
    assert _emu(L, lay, 32)[0] == 0
