"""CPU emulation of the GPU's floor-1 evaluation (tests/emu/floor1_emu.cpp compiles
lewton_b200/csrc/floor1_eval.cuh for the host): post unwrap + closed-form curve + DDA segment render +
the packed segments of k_prologue_fused against the oracle's literal restatement of audio.rs:391-555, on random floors incl. wild post values,
posts beyond n/2 and early-ending x lists."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import random_floor1, random_floor1_y

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "emu", "liblwb_floor1_emu.so")


def build():
    src = os.path.join(HERE, "emu", "floor1_emu.cpp")
    deps = [src] + [os.path.join(HERE, "..", "lewton_b200", "csrc", f) for f in ("floor1_eval.cuh", "tables_host.cpp", "lwb_common.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-I",
                               os.path.join(HERE, "..", "include"), "-o", SO, src])
    return SO


@pytest.mark.parametrize("seed", range(8))
def test_floor1_posts_closed_form_dda_and_packed_segments_match_the_oracle(oracle, seed):
    L = C.CDLL(build())
    rng = np.random.default_rng(1000 + seed)
    for case in range(150):
        n2 = int(rng.choice([32, 128, 512, 1024, 4096]))
        mult, xs = random_floor1(rng, n2)
        y = random_floor1_y(rng, mult, len(xs), wild=(case % 5 == 0))
        fl = oracle.make_floor1(mult, xs)
        final_y, step2 = oracle.floor1_amplitude(fl, y)
        want = np.asarray(oracle.floor1_curve_y(fl, final_y, step2, n2), np.uint32)
        xa, ya = np.array(xs, np.uint32), np.array(y, np.uint32)
        closed = np.zeros(n2, np.uint32)
        render = np.zeros(n2, np.uint8)
        packed = np.zeros(n2, np.uint8)
        rc = L.lwb_emu_floor1(mult, xa.ctypes.data_as(C.c_void_p), len(xs), ya.ctypes.data_as(C.c_void_p), n2,
                              closed.ctypes.data_as(C.c_void_p), render.ctypes.data_as(C.c_void_p),
                              packed.ctypes.data_as(C.c_void_p))
        assert rc == 0
        assert np.array_equal(packed.astype(np.uint32), want & 255), (seed, case, np.nonzero(packed != (want & 255))[0][:5])
        assert np.array_equal(closed & 255, want & 255), (seed, case)
        assert np.array_equal(render.astype(np.uint32), want & 255), (seed, case, np.nonzero(render != (want & 255))[0][:5])


def test_packed_segment_multiply_high_division_is_exact():
    """d_floor1_magic / d_mulhi_u32, the division d_floor1_pack_segment packs into each segment for k_prologue_fused,
    == integer division for every segment length it is used for."""
    L = C.CDLL(build())
    L.lwb_emu_magic_mismatches.restype = C.c_long
    assert L.lwb_emu_magic_mismatches(1, 32768) == 0
