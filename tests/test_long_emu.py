"""CPU emulation of the fused long-block kernel (tests/emu/long_emu.cpp): the kernel's per-lane
phase functions, element maps, swizzle and twiddle pack -- the same source the GPU compiles --
run lane by lane on the host and must reproduce the oracle bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
EMU_SO = os.path.join(EMU_DIR, "liblwb_emu.so")


def build_emu():
    src = os.path.join(EMU_DIR, "long_emu.cpp")
    hdr = os.path.join(HERE, "..", "lewton_b200", "csrc", "kernel_long.cuh")
    if (not os.path.exists(EMU_SO) or os.path.getmtime(EMU_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr))):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared",
                               "-o", EMU_SO, src])
    return EMU_SO


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(build_emu())
    vp = C.c_void_p
    L.lwb_emu_build_pack.argtypes = [vp] * 5
    L.lwb_emu_long_run.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    L.lwb_emu_long_run2.argtypes = [vp, vp, C.c_int, vp, vp, vp]
    return L


def P(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def pack(emu, oracle):
    t = oracle.tables(11)
    pk = np.zeros(emu.lwb_emu_pack_floats(), np.float32)
    emu.lwb_emu_build_pack(P(t.a), P(t.b), P(t.c), P(t.window), P(pk))
    return pk


def oracle_run(oracle, spec, state):
    pwr = oracle.Pwr(1, 11)
    if state is not None:
        pwr.set_data(state[None, :])
    outs = []
    for p in range(spec.shape[0]):
        rc, pcm = oracle.synth_spectrum(8, 11, 1, 1, 1, spec[p:p + 1], pwr)
        assert rc == 0
        outs.append(pcm[0])
    return np.concatenate(outs), pwr.data()[0]


@pytest.mark.parametrize("seed,npk,with_state,scale", [(0, 5, False, 1.0), (1, 1, False, 1.0), (2, 4, True, 1.0),
                                                       (3, 1, True, 1e-2), (4, 3, True, 1e-30), (5, 2, False, 1e30)])
def test_emulated_kernel_matches_oracle(emu, pack, oracle, seed, npk, with_state, scale):
    rng = np.random.default_rng(seed)
    spec = (rng.standard_normal((npk, 1024)) * scale).astype(np.float32)
    state = (rng.standard_normal(1024) * scale).astype(np.float32) if with_state else None   # NOT symmetric
    want, want_state = oracle_run(oracle, spec, state)
    st = state.copy() if with_state else np.zeros(1024, np.float32)
    out = np.zeros((npk, 1024), np.float32)
    conflicts = emu.lwb_emu_long_run(P(pack), P(spec), npk, int(with_state), P(st), P(out))
    assert conflicts == 1, "shared-memory transposes must be bank-conflict free"
    emitted = npk if with_state else npk - 1
    got = out[:emitted].ravel()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(st.view(np.uint32), want_state.view(np.uint32))


def test_emulated_kernel_special_values(emu, pack, oracle):
    """inf/NaN/denormal/zero inputs flow through identically (denormals are kept, not flushed)."""
    rng = np.random.default_rng(9)
    spec = rng.standard_normal((3, 1024)).astype(np.float32)
    spec[0, :64] = 1e-42          # denormals
    spec[1, 5] = np.inf
    spec[1, 77] = np.nan
    spec[2] = 0.0
    want, want_state = oracle_run(oracle, spec, None)
    st = np.zeros(1024, np.float32)
    out = np.zeros((3, 1024), np.float32)
    emu.lwb_emu_long_run(P(pack), P(spec), 3, 0, P(st), P(out))
    got = out[:2].ravel()
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    assert np.all(same)


@pytest.mark.parametrize("seed,npk,prev", [(20, 4, (0, 0)), (21, 3, (1, 0)), (22, 1, (0, 1)), (23, 5, (1, 1))])
def test_emulated_dual_block_matches_oracle(emu, pack, oracle, seed, npk, prev):
    """NB = 2: a warp transforms two runs in lockstep (LWB_LONG_NB=2; the shipped configuration is NB = 1)."""
    rng = np.random.default_rng(seed)
    spec = rng.standard_normal((2, npk, 1024)).astype(np.float32)
    states = rng.standard_normal((2, 1024)).astype(np.float32)
    st = states.copy()
    out = np.zeros((2, npk, 1024), np.float32)
    hp = np.array(prev, np.int32)
    conflicts = emu.lwb_emu_long_run2(P(pack), P(spec), npk, P(hp), P(st), P(out))
    assert conflicts == 1
    for b in range(2):
        want, want_state = oracle_run(oracle, spec[b], states[b] if prev[b] else None)
        emitted = npk if prev[b] else npk - 1
        got = out[b, :emitted].ravel()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), b
        assert np.array_equal(st[b].view(np.uint32), want_state.view(np.uint32)), b
