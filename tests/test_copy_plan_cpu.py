"""The PCM copy-back planner of the host-memory batch paths (lewton_b200/csrc/pcm_copy_plan.h, compiled for the host by
tests/emu/copy_plan_emu.cpp): on random layouts its copies cover every element of the chains' write set exactly once and
nothing else, and the layouts a decode server uses cost one copy."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import write_set
from lewton_b200 import _cabi as cabi

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "emu", "liblwb_copy_plan_emu.so")


def build():
    src = os.path.join(HERE, "emu", "copy_plan_emu.cpp")
    deps = [src, os.path.join(HERE, "..", "lewton_b200", "csrc", "pcm_copy_plan.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SO, src])
    return SO


class _Chain:
    def __init__(self, out_offset, out_stride, n_samples):
        self.out_offset, self.out_stride, self.n_samples = out_offset, out_stride, n_samples


def plan(chans, chains, fmt, max_pitch=1 << 40):
    lib = C.CDLL(build())
    lib.lwb_emu_copy_plan.restype = C.c_long
    n = len(chains)
    ch = np.array(chans, np.uint32)
    oo = np.array([c.out_offset for c in chains], np.uint64)
    st = np.array([c.out_stride for c in chains], np.uint64)
    ns = np.array([c.n_samples for c in chains], np.uint32)
    cap = max(1, sum(chans) + n)
    out = np.zeros((cap, 4), np.uint64)
    planar = int(fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR))
    k = lib.lwb_emu_copy_plan(planar, C.c_size_t(n), ch.ctypes.data_as(C.c_void_p), oo.ctypes.data_as(C.c_void_p),
                              st.ctypes.data_as(C.c_void_p), ns.ctypes.data_as(C.c_void_p), C.c_uint64(max_pitch),
                              out.ctypes.data_as(C.c_void_p), C.c_size_t(cap))
    assert k >= 0
    return [tuple(int(v) for v in row) for row in out[:k]]


def check_exact_cover(chans, chains, fmt, copies, max_pitch=1 << 40):
    ws = write_set(chains, lambda i: chans[i], fmt)
    size = max([s + n for _, spans in ws for s, n in spans] + [1])
    want = np.zeros(size, np.int32)
    for _, spans in ws:
        for s, n in spans:
            want[s:s + n] = 1
    got = np.zeros(size + 1, np.int32)
    for off, width, pitch, height in copies:
        assert width > 0 and height > 0
        assert height == 1 or width <= pitch <= max_pitch
        for r in range(height):
            assert off + r * pitch + width <= size, "a copy reaches past the write set"
            got[off + r * pitch:off + r * pitch + width] += 1
    assert got[size] == 0
    bad = np.nonzero(got[:size] != want)[0]
    assert bad.size == 0, f"element {bad[0]} copied {got[bad[0]]} times, in the write set: {bool(want[bad[0]])}"


def random_layout(rng):
    S = int(rng.integers(1, 24))
    chans = [int(rng.choice([1, 2, 3, 6, 8])) for _ in range(S)]
    ns = [int(rng.choice([0, 0, 1, 3, 128, 1024, int(rng.integers(1, 3000))])) for _ in range(S)]
    kind = rng.choice(["tight", "padded", "channel_major", "reverse", "odd", "interleaved"])
    fmt = cabi.OUT_F32_INTERLEAVED if kind == "interleaved" else cabi.OUT_F32_PLANAR
    stride = max(ns) + int(rng.integers(0, 9)) if kind != "tight" else max(ns)
    stride = max(stride, 1)
    chains, pos = [], int(rng.integers(0, 7))
    if kind == "channel_major":
        Cmax = max(chans)
        for s in range(S):
            chains.append(_Chain(pos + s * stride, S * stride, ns[s]))
        chans = [Cmax] * S if rng.random() < 0.5 else chans
    else:
        # odd: every chain its own stride and gap, so that offsets fall on any residue mod 4
        strides = [max(n, 1) + int(rng.integers(0, 4)) if kind == "odd" else stride for n in ns]
        chains = [_Chain(0, strides[s], ns[s]) for s in range(S)]
        for s in (range(S - 1, -1, -1) if kind == "reverse" else range(S)):
            chains[s].out_offset = pos
            pos += ns[s] * chans[s] if fmt == cabi.OUT_F32_INTERLEAVED else strides[s] * chans[s]
            if kind in ("padded", "odd", "interleaved"):
                pos += int(rng.integers(0, 5))
    return chans, chains, fmt


@pytest.mark.parametrize("seed", range(6))
def test_copies_cover_exactly_the_write_set(seed):
    rng = np.random.default_rng(900 + seed)
    for _ in range(150):
        chans, chains, fmt = random_layout(rng)
        max_pitch = int(rng.choice([1 << 40, 2048, 700]))
        check_exact_cover(chans, chains, fmt, plan(chans, chains, fmt, max_pitch), max_pitch)


def test_bench_layouts_cost_one_copy():
    S, C, stride = 64, 2, 16 * 1024
    # steady state: chains adjacent, out_stride == n_samples -> one contiguous copy
    tight = [_Chain(s * C * stride, stride, stride) for s in range(S)]
    assert plan([C] * S, tight, cabi.OUT_F32_PLANAR) == [(0, S * C * stride, S * C * stride, 1)]
    # first step of fresh streams: n_samples = stride - 1024 in every plane -> one 2D copy
    first = [_Chain(s * C * stride, stride, stride - 1024) for s in range(S)]
    assert plan([C] * S, first, cabi.OUT_F32_PLANAR) == [(0, stride - 1024, stride, S * C)]
    # one padded planar chain: one 2D copy of C rows
    assert plan([6], [_Chain(12, 5000, 4000)], cabi.OUT_I16_PLANAR) == [(12, 4000, 5000, 6)]
    # channel-major planes of equal-length chains interleave into one contiguous span
    cm = [_Chain(s * 300, S * 300, 300) for s in range(S)]
    assert plan([C] * S, cm, cabi.OUT_F32_PLANAR) == [(0, S * C * 300, S * C * 300, 1)]
    # nothing produced: no copy
    assert plan([2, 2], [_Chain(0, 8, 0), _Chain(16, 8, 0)], cabi.OUT_F32_PLANAR) == []


def test_pitch_limit_splits_a_2d_copy():
    chains = [_Chain(0, 5000, 100)]
    assert plan([4], chains, cabi.OUT_F32_PLANAR, max_pitch=4999) == [(k * 5000, 100, 100, 1) for k in range(4)]
    check_exact_cover([4], chains, cabi.OUT_F32_PLANAR, plan([4], chains, cabi.OUT_F32_PLANAR, max_pitch=4999), 4999)
