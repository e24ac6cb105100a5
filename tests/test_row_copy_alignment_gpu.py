"""k_row_copy at every shift class, head length and tail length, through the two features that use it with arbitrary
addresses: the samples of clipped chains (output windows) and lwb_streams_save / lwb_streams_load.

The cases come from tests/row_copy_cases.py, which computes the class of every row a batch or a state call copies --
its source-destination phase mod 16, head, 16-byte lines and tail -- from the layout the library gives it, and each
test first asserts that its rows reach every class (row_copy_cases.classes): all phases, heads and tails of the
element size, rows shorter than their head, rows of exactly one line, long rows, and chains or slots with no row.

Windowed batches are checked against their unwindowed twins (same setup, same packets): the written samples equal the
twin's decode sliced to the window (f32: also the oracle's, bit for bit), every element outside them keeps its
sentinel, and the windowed batch launches exactly the twin's kernels plus one k_row_copy.  A second layout packs the
rows with no padding (out_stride == written, chains back to back), so a store past the end of a row would show as a
wrong value in the next row rather than as a changed sentinel."""
import numpy as np
import pytest

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import ALL_KERNELS, bits_equal, expect_kernels, launches_are_attributed, make_setup
import row_copy_cases as R
from test_stream_windows_gpu import (DTYPE, F16I, F16P, F32I, F32P, FLOOR, I16I, I16P, PATHS, PLANAR, SPECTRUM, Arena, Batch, Stream,
                                     check_batch, check_oracle_and_states, decode, deinterleave)

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
FORMATS = [F32P, I16P, F16P, F32I, I16I, F16I]
FMT_IDS = ["f32p", "i16p", "f16p", "f32i", "i16i", "f16i"]
PACKETS = 3                  # long blocks per chain on fresh streams: 2 * 1024 samples
N = 2048
MIX = np.array([[0.5, 0.5], [0.0, 1.0], [1.0, 0.0]], np.float32)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 1: clipped chains
# ---------------------------------------------------------------------------------------------------------------------
def window_streams(ctx, oracle, fmt):
    """Stereo streams of the k_long shape, one per window of row_copy_cases.windows; interleaved batches give every
    fourth one a 3-channel output mix, so that skip * K and the chains' lengths are odd."""
    C, bs0, bs1, _, _, _ = PATHS["k_long"]
    mapping = [{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}]
    su = make_setup(ctx, C, bs0, bs1, mappings=mapping, floors=[FLOOR])
    mixed = None
    if fmt not in PLANAR:
        mixed = make_setup(ctx, C, bs0, bs1, mappings=mapping, floors=[FLOOR])
        mixed.set_output_mix(MIX)
    esz = np.dtype(DTYPE[fmt]).itemsize
    wins = R.windows(N, R.LINE // esz // (1 if fmt in PLANAR else C))
    with_oracle = oracle if fmt in (F32P, F32I) else None
    out = []
    for j, w in enumerate(wins):
        s = mixed if mixed is not None and j % 4 == 2 else su
        out.append(Stream(s, with_oracle if s is su else None, C, bs0, bs1, np.ones(PACKETS, np.uint8), w))
    return out


@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("base", [0, 1], ids=["base0", "base1"])
@pytest.mark.parametrize("memory", [DEVICE, HOST], ids=["device", "host"])
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_clipped_rows_at_every_class(ctx, oracle, fmt, memory, base, packed):
    """One batch of ~100 windowed chains whose rows reach every class, in an arena `base` elements past a 16-byte
    boundary (host memory: the kernel sees the staging, whose phase is the element offsets').  The twin's arena has the
    same base: a device-memory batch keeps its clipped chains' scratch at the base's phase, so the twin and the
    windowed batch take one path -- k_long for planar output on an aligned base, else the chain kernel."""
    rng = np.random.default_rng(100 + 10 * FORMATS.index(fmt) + 4 * memory + 2 * base + packed)
    planar, esz = fmt in PLANAR, np.dtype(DTYPE[fmt]).itemsize
    streams = window_streams(ctx, oracle, fmt)
    b = Batch(rng, streams, PACKETS, SPECTRUM, fmt)
    assert all(p[7] == N for p in b.parts)
    base_byte = 0 if memory == HOST else base * esz
    lay, size = R.layout([st.window for st in streams], N, b.K, planar, packed, start=((-base_byte) % R.LINE) // esz)
    b.win_lay, b.win_elems = lay, size
    rows, empty = R.window_rows([st.window for st in streams], lay, N, b.K, planar, esz, base_byte)
    assert not R.missing(rows, esz, empty), R.missing(rows, esz, empty)

    fa = Arena(ctx, b.full_elems, fmt, memory, shift=base * esz)
    wa = Arena(ctx, b.win_elems, fmt, memory, shift=base * esz)
    if memory == DEVICE:
        assert wa.ptr % R.LINE == base_byte
    fch, wch = b.chains("full", b.full_lay), b.chains("win", b.win_lay)
    with expect_kernels(ctx) as kfull:
        decode(ctx, b, "full", memory, fa, fch)
    with expect_kernels(ctx) as kwin:
        decode(ctx, b, "win", memory, wa, wch)
    fbuf, wbuf = fa.read(), wa.read()
    written = check_batch(b, fch, wch, fbuf, wbuf)
    assert written == [R.clip(st.window, N)[1] for st in streams]
    assert kfull["k_long" if planar and not base_byte else "k_chain"] > 0, kfull
    want = dict(kfull)
    want["k_row_copy"] += 1
    assert kwin == want, (kfull, kwin)
    full_pcm = [deinterleave(fbuf.view(DTYPE[fmt])[o:], fmt, K, N).astype(np.float32) for (o, _), K in zip(b.full_lay, b.K)]
    check_oracle_and_states(streams, full_pcm, fmt)


# ---------------------------------------------------------------------------------------------------------------------
# 2: lwb_streams_save / lwb_streams_load
# ---------------------------------------------------------------------------------------------------------------------
ROW_COPY_ONLY = dict(ran={"k_row_copy": 1}, not_ran=ALL_KERNELS - {"k_row_copy"})
FILL = -7.0


class StateBuffer:
    """n floats of page-locked host memory or device memory, `base` floats past a 16-byte boundary, filled with FILL."""

    def __init__(self, ctx, memory, n, base):
        import torch
        self.memory, self.base, self.n = memory, base, n
        if memory == HOST:
            self.h = ctx.host_alloc(n + 8, np.float32)
            assert self.h.ctypes.data % R.LINE == 0
            self.h[...] = FILL
            self.ptr = self.h[base:base + n]
        else:
            self.t = torch.full((n + 8,), FILL, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            assert self.t.data_ptr() % R.LINE == 0
            self.ptr = self.t.data_ptr() + 4 * base

    def read(self):
        """The whole allocation, the margins around the buffer included."""
        return np.array(self.h) if self.memory == HOST else self.t.cpu().numpy()


@pytest.mark.parametrize("gap", [0, 1], ids=["back_to_back", "gaps"])
@pytest.mark.parametrize("base", range(4), ids=[f"base{b}" for b in range(4)])
@pytest.mark.parametrize("memory", [DEVICE, HOST], ids=["device", "host"])
def test_state_rows_at_every_class(ctx, memory, base, gap):
    """Streams with states of every length of row_copy_cases.state_lengths, saved to and loaded from slots at every
    residue mod 4: the saved rows are export_state's bit for bit, every element outside the slots keeps its fill, and
    after a load into other streams (holding other states) export_state gives the rows back."""
    rng = np.random.default_rng(200 + 8 * memory + 2 * base + gap)
    C, bs0, bs1 = 2, 8, 11
    su = make_setup(ctx, C, bs0, bs1, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=[FLOOR])
    slots_at, size = R.state_slots(R.state_lengths(1 << bs1), C, gap)
    for load in (False, True):
        rows, empty = R.state_rows(slots_at, C, base, memory == HOST, load)
        want = R.load_classes() if load else R.classes(4)
        assert not R.missing(rows, 4, empty, want), (load, R.missing(rows, 4, empty, want))
    pwrs = []
    for _, n in slots_at:
        p = L.PreviousWindowRight(su)
        p.set_data(rng.standard_normal((C, n)).astype(np.float32))        # has = 1 at every length, 0 included
        pwrs.append(p)
    buf = StateBuffer(ctx, memory, size, base)
    with expect_kernels(ctx, **ROW_COPY_ONLY):
        slots, t = ctx.save_states(pwrs, buf.ptr, memory, [o for o, _ in slots_at])
        t.wait()
    got = buf.read()
    inside = np.zeros(got.size, bool)
    for p, s, (o, n) in zip(pwrs, slots, slots_at):
        assert (s.has, s.len, s.offset) == (True, n, o)
        a = base + o
        assert bits_equal(got[a:a + C * n].reshape(C, n), p.data() if n else np.zeros((C, 0))), (o, n)
        inside[a:a + C * n] = True
    assert np.all(got[~inside] == FILL), f"a save wrote outside its slots: {np.nonzero(got[~inside] != FILL)[0][:8]}"
    fresh = []
    for p in pwrs:
        f = L.PreviousWindowRight(su)
        f.set_data(np.full((C, 64), 3.0, np.float32))
        fresh.append(f)
    with expect_kernels(ctx, **ROW_COPY_ONLY):
        ctx.load_states([L.StateSlot(f, s.offset, s.len, s.has) for f, s in zip(fresh, slots)], buf.ptr, memory).wait()
    for f, p, (o, n) in zip(fresh, pwrs, slots_at):
        assert not f.is_empty() and len(f) == n, (o, n, len(f))
        if n:
            assert bits_equal(f.data(), p.data()), (o, n)
    assert np.array_equal(buf.read().view(np.uint32), got.view(np.uint32)), "a load wrote to its buffer"
