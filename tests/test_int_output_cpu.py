"""The i32 and packed i24 output formats without a GPU: the header's values (6 and 7 unassigned), the Python constants,
the unchanged ABI, and the integer references the GPU tests hold the kernels to (numpy: an f32 multiply by 2^31 / 2^23,
truncation toward zero, saturation, NaN -> 0), checked against exact integer arithmetic on the f32 bit patterns."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from lewton_b200 import _cabi
from lewton_b200.api import I24, i24_to_i32, sample_format
from test_f16_output_cpu import ROOT, _compile_and_run

I32_SCALE, I24_SCALE = np.float32(2.0 ** 31), np.float32(2.0 ** 23)
I24_MIN, I24_MAX = -(1 << 23), (1 << 23) - 1


def int_test_values():
    """float32 values at every edge of the two rules (also what test_int_output_gpu feeds each store site): +-0, +-1.0 and
    their neighbours, every clamp edge of both scales and one ulp either side, values that scale to integers and to
    integers +- 1/2 and +- one ulp, f32 subnormals, +-inf, quiet and signalling NaNs, and random f32 bit patterns."""
    f32 = np.float32
    one = np.array([0.0, 1.0, 0.5, 0.25, 2.0, 1e-3, 3e5, 1e30, 3.4e38], f32)
    # i24 edges: 8388607.x / 2^23, -8388608 / 2^23 = -1, -8388609 / 2^23; i32 edges: +-2^31 / 2^31 = +-1
    edges = np.array([I24_MAX / 2 ** 23, (I24_MAX + 0.5) / 2 ** 23, (I24_MAX + 1) / 2 ** 23, (I24_MIN - 1) / 2 ** 23,
                      (I24_MIN - 0.5) / 2 ** 23, I24_MIN / 2 ** 23, 1 - 2 ** -24, 1 - 2 ** -23, 2 ** -31, 2 ** -23, 2 ** -24], np.float64).astype(f32)
    base = np.concatenate([one, edges])
    base = np.concatenate([base, np.nextafter(base, f32(np.inf)), np.nextafter(base, f32(-np.inf))])
    base = np.concatenate([base, -base, np.array([-0.0, np.inf, -np.inf], f32)])
    rng = np.random.default_rng(24)
    k = rng.integers(-(1 << 23), 1 << 23, 2048)
    ints = np.concatenate([k / 2 ** 23, (k + 0.5) / 2 ** 23, (k.astype(np.int64) << 8) / 2 ** 31]).astype(f32)
    ints = np.concatenate([ints, np.nextafter(ints, f32(np.inf)), np.nextafter(ints, f32(-np.inf))])
    nans = np.array([0x7fc00000, 0xffc00000, 0x7fc12345, 0x7f800001, 0xff800001, 0x7fa5a5a5, 0x7fffffff], np.uint32).view(f32)
    sub = np.array([1, 2, 3, 0x7fffff, 0x400000, 0x12345], np.uint32).view(f32)
    bits = rng.integers(0, 1 << 32, 8192, dtype=np.uint64).astype(np.uint32).view(f32)
    small = (rng.standard_normal(4096) * 0.3).astype(f32)                      # where decoded audio lives
    return np.concatenate([base, ints, nans, sub, -sub, bits, small]).astype(f32)


def _to_int(v, scale, lo, hi):
    with np.errstate(over="ignore", invalid="ignore"):
        y = np.asarray(v, np.float32) * scale                                   # one f32 multiply, exact
        t = np.trunc(y.astype(np.float64))
        out = np.where(np.isnan(t), 0, np.clip(np.nan_to_num(t, nan=0.0, posinf=hi, neginf=lo), lo, hi))
    return out.astype(np.int64)


def to_i32(v):
    """The I32 rule: int32 of v * 2^31, truncated toward zero, saturated (1.0 -> INT32_MAX), NaN -> 0."""
    return _to_int(v, I32_SCALE, -(1 << 31), (1 << 31) - 1).astype(np.int32)


def to_i24(v):
    """The I24 rule as int32 values in [-2^23, 2^23): v * 2^23 truncated toward zero, saturated, NaN -> 0."""
    return _to_int(v, I24_SCALE, I24_MIN, I24_MAX).astype(np.int32)


def pack_i24(ints):
    """int32 values in the i24 range -> I24 elements (the low 3 bytes, little-endian)."""
    a = np.ascontiguousarray(ints, np.int32)
    return np.ascontiguousarray(a.view(np.uint8).reshape(a.shape + (4,))[..., :3]).view(I24).reshape(a.shape)


def _exact(bits, shift, lo, hi):
    """trunc(x * 2^shift) saturated to [lo, hi], NaN -> 0, from the f32 bit pattern with Python integers only."""
    b = int(bits)
    sign, e, m = b >> 31, (b >> 23) & 0xff, b & 0x7fffff
    if e == 0xff:
        return 0 if m else (lo if sign else hi)
    mant, exp = (m, -149) if e == 0 else (m | 0x800000, e - 150)              # x = mant * 2^exp
    exp += shift
    mag = mant << exp if exp >= 0 else mant >> -exp                          # truncation toward zero of |x| 2^shift
    val = -mag if sign else mag
    return max(lo, min(hi, val))


def test_header_values_and_python_constants(tmp_path):
    got = _compile_and_run(tmp_path, 'printf("%d %d %d %d %d\\n", LWB_OUT_I32_PLANAR, LWB_OUT_I32_INTERLEAVED, '
                                     "LWB_OUT_I24_PLANAR, LWB_OUT_I24_INTERLEAVED, LWB_ABI_VERSION);")
    assert got == [8, 9, 10, 11, 3]
    assert (_cabi.OUT_I32_PLANAR, _cabi.OUT_I32_INTERLEAVED, _cabi.OUT_I24_PLANAR, _cabi.OUT_I24_INTERLEAVED) == tuple(got[:4])
    # 6 and 7 stay unassigned: no LWB_OUT_* name and no Python constant has them
    header = open(os.path.join(ROOT, "include", "lewton_b200.h")).read()
    assert "= 6" not in header.split("LWB_OUT_F32_PLANAR = 0")[1].split("};")[0]
    assert "= 7" not in header.split("LWB_OUT_F32_PLANAR = 0")[1].split("};")[0]
    values = {getattr(_cabi, n) for n in dir(_cabi) if n.startswith("OUT_")}
    assert values == {0, 1, 2, 3, 4, 5, 8, 9, 10, 11}


def test_struct_sizes_unchanged(tmp_path):
    """ABI 3's structs, as the C compiler sees them, still match the ctypes mirror: i32 and i24 added no field."""
    got = _compile_and_run(tmp_path, 'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(lwb_tables_ref), '
                                     "sizeof(lwb_floor_desc), sizeof(lwb_mapping_desc), sizeof(lwb_mode_desc), "
                                     "sizeof(lwb_setup_desc), sizeof(lwb_packet), sizeof(lwb_chain), sizeof(lwb_batch_io), "
                                     "sizeof(lwb_codebook_desc), sizeof(lwb_residue_desc), sizeof(lwb_vq_run));")
    want = [C.sizeof(t) for t in (_cabi.TablesRef, _cabi.FloorDesc, _cabi.MappingDesc, _cabi.ModeDesc, _cabi.SetupDesc,
                                  _cabi.Packet, _cabi.Chain, _cabi.BatchIo, _cabi.CodebookDesc, _cabi.ResidueDesc, _cabi.VqRun)]
    assert got == want


def test_sample_format_table():
    assert sample_format("i32") == (_cabi.OUT_I32_PLANAR, np.int32)
    assert sample_format("i32", True) == (_cabi.OUT_I32_INTERLEAVED, np.int32)
    assert sample_format("i24") == (_cabi.OUT_I24_PLANAR, I24)
    assert sample_format("i24", True) == (_cabi.OUT_I24_INTERLEAVED, I24)
    assert I24.itemsize == 3
    with pytest.raises(KeyError):
        sample_format("s24")


def test_value_set_covers_the_edges():
    v = int_test_values()
    assert np.isnan(v).sum() >= 7 and np.isposinf(v).any() and np.isneginf(v).any()
    assert ((np.abs(v) > 0) & (np.abs(v) < np.finfo(np.float32).tiny)).any()
    assert (v == 1.0).any() and (v == -1.0).any() and (v == np.nextafter(np.float32(1), np.float32(0))).any()
    assert (np.signbit(v) & (v == 0)).any() and (~np.signbit(v) & (v == 0)).any()
    i24 = to_i24(v)
    for e in (I24_MAX, I24_MIN, I24_MAX - 1, I24_MIN + 1):
        assert (i24 == e).any(), e
    i32 = to_i32(v)
    assert (i32 == 2 ** 31 - 1).any() and (i32 == -2 ** 31).any() and (i32 == 0).sum() > 8


@pytest.mark.parametrize("rule,shift,lo,hi", [(to_i32, 31, -(1 << 31), (1 << 31) - 1), (to_i24, 23, I24_MIN, I24_MAX)])
def test_reference_matches_exact_integer_arithmetic(rule, shift, lo, hi):
    v = int_test_values()
    got = rule(v)
    want = np.array([_exact(b, shift, lo, hi) for b in v.view(np.uint32)], np.int64)
    bad = np.nonzero(got.astype(np.int64) != want)[0]
    assert not bad.size, (bad[:4], v[bad[:4]], got[bad[:4]], want[bad[:4]])
    assert rule(np.float32(1.0)) == hi and rule(np.float32(-1.0)) == (lo if shift == 31 else -(1 << 23))


def test_i24_widening():
    v = int_test_values()
    ints = to_i24(v)
    packed = pack_i24(ints)
    assert packed.dtype == I24 and packed.shape == ints.shape
    assert np.array_equal(i24_to_i32(packed), ints)
    raw = packed.view(np.uint8)
    assert np.array_equal(raw[0::3].astype(np.int64) | raw[1::3].astype(np.int64) << 8 | raw[2::3].astype(np.int64) << 16,
                          ints.astype(np.int64) & 0xffffff)
    assert np.array_equal(i24_to_i32(raw.reshape(-1, 6)), ints.reshape(-1, 2))           # uint8, 3 bytes per sample
    t = torch.from_numpy(raw.copy())
    assert np.array_equal(i24_to_i32(t).numpy(), ints)
    with pytest.raises(ValueError):
        i24_to_i32(np.zeros(4, np.uint8))
