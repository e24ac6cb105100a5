"""The case generators of the k_row_copy tests (tests/row_copy_cases.py) reach every class of row, without a GPU: every
phase, head and tail for each element size, rows shorter than their head, rows of one 16-byte line, long rows and
chains or slots with no row -- in every output format, memory space, PCM base and layout the GPU tests run, and for
saves and loads at every buffer base and slot spacing.  So a generator change that loses a class fails here."""
import pytest

import row_copy_cases as R

N = 2048
FORMATS = {"f32p": (4, True), "i16p": (2, True), "f16p": (2, True), "f32i": (4, False), "i16i": (2, False), "f16i": (2, False)}


def test_split_matches_the_kernels_arithmetic():
    # (dst byte mod 16, bytes) -> (head, lines, tail): head up to the next boundary, or the whole row if shorter
    cases = {(0, 16): (0, 1, 0), (0, 2): (0, 0, 2), (2, 2): (2, 0, 0), (2, 14): (14, 0, 0), (2, 16): (14, 0, 2),
             (4, 44): (12, 2, 0), (14, 50): (2, 3, 0), (8, 0): (0, 0, 0), (12, 4): (4, 0, 0), (12, 40): (4, 2, 4)}
    for (d, n), want in cases.items():
        assert R.split(d, n) == want, (d, n)
    assert R.Row(6, 2, 32, 2).phase == 4 and R.Row(2, 6, 32, 2).phase == 12


@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("base", [0, 1], ids=["base0", "base1"])
@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_window_cases_reach_every_class(fmt, host, base, packed):
    esz, planar = FORMATS[fmt]
    wins = R.windows(N, R.LINE // esz // (1 if planar else 2))
    Ks = [2] * len(wins) if planar else [3 if j % 4 == 2 else 2 for j in range(len(wins))]
    base_byte = 0 if host else base * esz
    lay, size = R.layout(wins, N, Ks, planar, packed, start=((-base_byte) % R.LINE) // esz)
    rows, empty = R.window_rows(wins, lay, N, Ks, planar, esz, base_byte)
    assert not R.missing(rows, esz, empty)
    # every window clips its chain (the batch keeps its unwindowed path) and the layout stays inside the arena
    assert all(R.clip(w, N) != (0, N) for w in wins)
    for (off, stride), w, K in zip(lay, wins, Ks):
        written = R.clip(w, N)[1]
        end = off + ((K - 1) * stride + written if planar else K * written)
        assert end <= size
        if packed and planar:
            assert stride == written
    if packed:          # back to back: each chain starts where the one before ends
        for (o0, _), (o1, _), w, K in zip(lay, lay[1:], wins, Ks):
            assert o1 == o0 + K * R.clip(w, N)[1]


@pytest.mark.parametrize("gap", [0, 1], ids=["back_to_back", "gaps"])
@pytest.mark.parametrize("base", range(4))
@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_state_cases_reach_every_class(host, base, gap):
    slots, size = R.state_slots(R.state_lengths(2048), 2, gap)
    assert {o % 4 for o, n in slots if n} == {0, 1, 2, 3}
    assert all(o + 2 * n <= size for o, n in slots)
    assert all(o0 + 2 * n0 <= o1 for (o0, n0), (o1, _) in zip(slots, slots[1:]))
    if gap:
        assert all(o0 + 2 * n0 < o1 for (o0, n0), (o1, _) in zip(slots, slots[1:]))
    for load in (False, True):
        rows, empty = R.state_rows(slots, 2, base, host, load)
        assert not R.missing(rows, 4, empty, R.load_classes() if load else None), load
