"""The f16 output formats without a GPU: the header's values, the Python constants, the unchanged ABI, and the f16
reference the GPU tests hold the kernels to (numpy's float32 -> float16), checked against a second, independent
round-to-nearest-even implementation (torch's CPU conversion) on every value the conversion tests feed the kernels.
(The g++ emulations of tests/emu include the edited kernel headers; test_long_emu / test_short_emu / test_mid_emu build
them.)"""
import os
import subprocess

import numpy as np
import pytest
import torch

from lewton_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def f16_test_values():
    """float32 values at every rounding boundary of float32 -> float16 (also what test_f16_output_gpu feeds each store
    site): every finite f16 value; the f32 midpoints between neighbouring f16 values and one f32 ulp either side of each;
    +-65504, +-65520 and their f32 neighbours; +-inf; quiet and signalling NaNs; f32 subnormals; the f16 subnormal range."""
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    h = np.sort(h[np.isfinite(h)].astype(np.float32))
    h = np.unique(h)                                                  # (+0 and -0 are one value here; -0 is added below)
    mid = ((h[:-1].astype(np.float64) + h[1:].astype(np.float64)) / 2).astype(np.float32)   # exact in f32
    up, down = np.nextafter(mid, np.float32(np.inf)), np.nextafter(mid, np.float32(-np.inf))
    edges = np.array([65504, 65520, 65536, 1e30, 3.4e38], np.float32)
    edges = np.concatenate([edges, np.nextafter(edges, np.float32(np.inf)), np.nextafter(edges, np.float32(0))])
    edges = np.concatenate([edges, -edges, np.array([np.inf, -np.inf, 0.0, -0.0], np.float32)])
    nans = np.array([0x7fc00000, 0xffc00000, 0x7fc12345, 0x7f800001, 0xff800001, 0x7fa5a5a5, 0x7fffffff], np.uint32).view(np.float32)
    sub32 = np.array([1, 2, 3, 0x7fffff, 0x400000, 0x12345], np.uint32).view(np.float32)
    sub32 = np.concatenate([sub32, -sub32])
    rng = np.random.default_rng(16)
    sub16 = (rng.random(4096) * 2 ** -14).astype(np.float32) * rng.choice(np.array([-1, 1], np.float32), 4096)
    return np.concatenate([h, mid, up, down, edges, nans, sub32, sub16]).astype(np.float32)


def to_f16(v):
    """numpy's float32 -> float16: round to nearest even, subnormals kept, overflow to inf (the f16 formats' rule)."""
    with np.errstate(over="ignore"):
        return np.asarray(v, np.float32).astype(np.float16)


def _compile_and_run(tmp_path, body):
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include "lewton_b200.h"\nint main(void){' + body + "return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def test_header_values_and_python_constants(tmp_path):
    got = _compile_and_run(tmp_path, 'printf("%d %d %d %d %d %d %d\\n", LWB_OUT_F32_PLANAR, LWB_OUT_I16_PLANAR, '
                                     "LWB_OUT_F32_INTERLEAVED, LWB_OUT_I16_INTERLEAVED, LWB_OUT_F16_PLANAR, "
                                     "LWB_OUT_F16_INTERLEAVED, LWB_ABI_VERSION);")
    assert got == [0, 1, 2, 3, 4, 5, 3]
    assert (_cabi.OUT_F32_PLANAR, _cabi.OUT_I16_PLANAR, _cabi.OUT_F32_INTERLEAVED, _cabi.OUT_I16_INTERLEAVED,
            _cabi.OUT_F16_PLANAR, _cabi.OUT_F16_INTERLEAVED) == tuple(got[:6])


def test_struct_sizes_unchanged(tmp_path):
    """ABI 3's structs, as the C compiler sees them, still match the ctypes mirror: f16 added no field."""
    got = _compile_and_run(tmp_path, 'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(lwb_tables_ref), '
                                     "sizeof(lwb_floor_desc), sizeof(lwb_mapping_desc), sizeof(lwb_mode_desc), "
                                     "sizeof(lwb_setup_desc), sizeof(lwb_packet), sizeof(lwb_chain), sizeof(lwb_batch_io), "
                                     "sizeof(lwb_codebook_desc), sizeof(lwb_residue_desc), sizeof(lwb_vq_run));")
    import ctypes as C
    want = [C.sizeof(t) for t in (_cabi.TablesRef, _cabi.FloorDesc, _cabi.MappingDesc, _cabi.ModeDesc, _cabi.SetupDesc,
                                  _cabi.Packet, _cabi.Chain, _cabi.BatchIo, _cabi.CodebookDesc, _cabi.ResidueDesc, _cabi.VqRun)]
    assert got == want


def test_sample_format_table():
    from lewton_b200.api import sample_format
    assert sample_format("f16") == (_cabi.OUT_F16_PLANAR, np.float16)
    assert sample_format("f16", True) == (_cabi.OUT_F16_INTERLEAVED, np.float16)
    assert sample_format("i16", True) == (_cabi.OUT_I16_INTERLEAVED, np.int16)
    with pytest.raises(KeyError):
        sample_format("bf16")


def test_value_set_covers_the_rounding_boundaries():
    v = f16_test_values()
    assert v.dtype == np.float32
    h = to_f16(v)
    finite16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    finite16 = finite16[np.isfinite(finite16)]
    # every finite f16 value is hit exactly, and ties, overflow, NaNs and subnormals are all present
    assert np.isin(finite16.view(np.uint16), h.view(np.uint16)).all()
    assert np.isinf(h).sum() >= 4 and np.isnan(v).sum() >= 4
    assert ((np.abs(v) > 0) & (np.abs(v) < np.finfo(np.float32).tiny)).any()      # f32 subnormals
    assert ((np.abs(h) > 0) & (np.abs(h) < np.finfo(np.float16).tiny)).any()      # f16 subnormals
    assert (v == 65520).any() and (v == -65520).any() and (v == 65504).any()


def test_numpy_and_torch_round_alike():
    """Two round-to-nearest-even conversions agree bit for bit (NaN: any NaN) before the GPU is held to one of them."""
    v = f16_test_values()
    a = to_f16(v)
    b = torch.from_numpy(v.copy()).to(torch.float16).numpy()
    nan = np.isnan(a) & np.isnan(b)
    assert np.isnan(a).sum() == np.isnan(v).sum()
    assert bool(np.all((a.view(np.uint16) == b.view(np.uint16)) | nan))
