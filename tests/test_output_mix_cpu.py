"""The output channel mix (lwb_setup_set_output_mix) without a GPU: the ABI stays 3 with the same structs and kernel ids,
the new entry points are exported, declared and refuse NULL, the Python helper matrices are right, and the numpy
restatement the GPU tests hold the kernels to (tests/mix_oracle.py) sums in the stated order."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import lewton_b200 as L
from lewton_b200 import _cabi
from mix_oracle import mix_f32
from test_f16_output_cpu import _compile_and_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIX = {"lwb_setup_set_output_mix": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_float)]),
       "lwb_setup_output_channels": (C.c_uint32, [C.c_void_p])}


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import build
    build.build()
    return _cabi.lib()


def test_abi_structs_and_kernel_ids_unchanged(tmp_path):
    got = _compile_and_run(tmp_path, 'printf("%d %d %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", LWB_ABI_VERSION, '
                                     "LWB_KERNEL_COUNT, sizeof(lwb_tables_ref), sizeof(lwb_floor_desc), sizeof(lwb_mapping_desc), "
                                     "sizeof(lwb_mode_desc), sizeof(lwb_setup_desc), sizeof(lwb_packet), sizeof(lwb_chain), "
                                     "sizeof(lwb_batch_io), sizeof(lwb_codebook_desc), sizeof(lwb_residue_desc), sizeof(lwb_vq_run));")
    want = [C.sizeof(t) for t in (_cabi.TablesRef, _cabi.FloorDesc, _cabi.MappingDesc, _cabi.ModeDesc, _cabi.SetupDesc,
                                  _cabi.Packet, _cabi.Chain, _cabi.BatchIo, _cabi.CodebookDesc, _cabi.ResidueDesc, _cabi.VqRun)]
    assert got == [3, 14] + want
    assert len(_cabi.KERNELS) == 14 and _cabi.KERNELS[6] == "k_chain" and _cabi.KERNELS[11] == "k_overlap"


def test_mix_symbols_exported_declared_and_typed(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_b200.h")).read(), flags=re.S)
    assert re.search(r"\bint\s+lwb_setup_set_output_mix\s*\(\s*lwb_setup\s*\*\s*setup\s*,\s*uint32_t\s+n_out\s*,\s*const\s+float\s*\*\s*matrix\s*\)", hdr)
    assert re.search(r"\buint32_t\s+lwb_setup_output_channels\s*\(\s*const\s+lwb_setup\s*\*\s*setup\s*\)", hdr)
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (lwb_[a-z0-9_]+)", nm))
    for name, (res, args) in MIX.items():
        assert name in exported, name
        assert _cabi.SYMBOLS[name][0] is res and _cabi.SYMBOLS[name][1] == args, name


def test_mix_entry_points_refuse_null(lib):
    m = (C.c_float * 2)(1.0, 1.0)
    assert lib.lwb_setup_set_output_mix(None, 1, m) == _cabi.ERR_INVALID
    assert lib.lwb_setup_set_output_mix(None, 0, None) == _cabi.ERR_INVALID
    assert lib.lwb_setup_output_channels(None) == 0


VORBIS = {1: ["M"], 2: ["L", "R"], 3: ["L", "C", "R"], 4: ["FL", "FR", "BL", "BR"], 5: ["FL", "FC", "FR", "BL", "BR"],
          6: ["FL", "FC", "FR", "BL", "BR", "LFE"], 7: ["FL", "FC", "FR", "SL", "SR", "BC", "LFE"],
          8: ["FL", "FC", "FR", "SL", "SR", "BL", "BR", "LFE"]}                          # Vorbis I section 4.3.9
WAV = {1: ["M"], 2: ["L", "R"], 3: ["L", "R", "C"], 4: ["FL", "FR", "BL", "BR"], 5: ["FL", "FR", "FC", "BL", "BR"],
       6: ["FL", "FR", "FC", "LFE", "BL", "BR"], 7: ["FL", "FR", "FC", "LFE", "BC", "SL", "SR"],
       8: ["FL", "FR", "FC", "LFE", "BL", "BR", "SL", "SR"]}                            # WAVEFORMATEXTENSIBLE mask order


@pytest.mark.parametrize("channels", range(1, 9))
def test_wav_order_matrices(channels):
    m = L.mix_wav_order(channels)
    assert m.dtype == np.float32 and m.shape == (channels, channels)
    assert np.array_equal(np.sort(m, axis=1)[:, -1], np.ones(channels)) and (m.sum(axis=1) == 1).all()
    assert (m.sum(axis=0) == 1).all()                                                  # a permutation
    names = np.array(VORBIS[channels])
    assert list(names[m.argmax(axis=1)]) == WAV[channels]


def test_mono_and_select_matrices():
    for c in (1, 2, 3, 6, 10, 255):
        m = L.mix_mono(c)
        assert m.dtype == np.float32 and m.shape == (1, c)
        assert (m.view(np.uint32) == (np.float32(1) / np.float32(c)).view(np.uint32)).all()
    s = L.mix_select(6, [0, 2, 2])
    assert s.dtype == np.float32 and s.tolist() == [[1, 0, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0], [0, 0, 1, 0, 0, 0]]
    with pytest.raises(ValueError):
        L.mix_select(2, [2])
    with pytest.raises(ValueError):
        L.mix_wav_order(9)


def test_numpy_mix_equals_float64_where_exact():
    """Small integers times powers of two: every product and partial sum is exact in f32, so the f32 mix equals the
    float64 matrix product."""
    rng = np.random.default_rng(7)
    for C_, K in ((2, 1), (6, 2), (8, 8), (1, 2), (10, 2)):
        x = rng.integers(-4096, 4097, (C_, 500)).astype(np.float32)
        m = (rng.integers(-4, 5, (K, C_)) * 2.0 ** rng.integers(-3, 3, (K, C_))).astype(np.float32)
        if K > 1:
            m[0] = 0                                                                   # an empty row
        got = mix_f32(x, m)
        want = m.astype(np.float64) @ x.astype(np.float64)
        assert got.dtype == np.float32 and np.array_equal(got.astype(np.float64), want), (C_, K)


def test_numpy_mix_order_and_signed_zero():
    x = np.array([[1e8], [1.0], [-1e8], [-0.0]], np.float32)
    # left to right in channel order: (1e8 + 1) - 1e8 = 0 in f32 (1e8 + 1 rounds to 1e8), (1e8 - 1e8) + 1 = 1
    assert mix_f32(x, [[1, 1, 1, 0]])[0, 0] == 0.0
    assert mix_f32(x[[0, 2, 1]], [[1, 1, 1]])[0, 0] == 1.0
    # the first term is not added to a zero: a single -0.0 stays -0.0; an empty row is +0.0
    y = mix_f32(x, [[0, 0, 0, 1], [0, 0, 0, 0]])
    assert np.signbit(y[0, 0]) and not np.signbit(y[1, 0])
    # one 1.0 copies its channel bit for bit, NaN payloads included
    z = np.array([[np.float32(3.5)], [np.array([0x7fc12345], np.uint32).view(np.float32)[0]]], np.float32)
    assert mix_f32(z, [[0, 1], [1, 0]]).view(np.uint32).tolist() == [[0x7fc12345], [np.float32(3.5).view(np.uint32)]]
