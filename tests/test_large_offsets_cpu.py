"""Host-side pieces of the large-offset tests (tests/test_large_offsets_gpu.py), without a GPU: the ctypes layouts of the
CUDA driver structs the sparse arenas pass to cuMemCreate / cuMemSetAccess, against cuda.h; the 32-bit images of a span
the arenas map as mirror windows; and the PCM copy-back planner of host-memory batches at offsets and pitches past
2^32."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import sparse_arena as sa
from lewton_b200 import _cabi as cabi
from test_copy_plan_cpu import _Chain, plan

F32P, F32I = cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED


def cuda_include():
    nvcc = shutil.which("nvcc")
    for root in ([os.path.dirname(os.path.dirname(nvcc))] if nvcc else []) + [os.environ.get("CUDA_HOME", ""), "/usr/local/cuda"]:
        if root and os.path.exists(os.path.join(root, "include", "cuda.h")):
            return os.path.join(root, "include")
    pytest.fail("cuda.h not found (nvcc on PATH, CUDA_HOME or /usr/local/cuda)")


LAYOUT_PROBE = r"""
#include <cuda.h>
#include <stddef.h>
#include <stdio.h>
#define F(T, f) printf(#T " " #f " %zu %zu\n", offsetof(T, f), sizeof(((T *)0)->f))
int main(void)
{
    printf("CUmemLocation - %zu %zu\n", sizeof(CUmemLocation), _Alignof(CUmemLocation));
    F(CUmemLocation, type); F(CUmemLocation, id);
    printf("CUmemAllocationProp - %zu %zu\n", sizeof(CUmemAllocationProp), _Alignof(CUmemAllocationProp));
    F(CUmemAllocationProp, type); F(CUmemAllocationProp, requestedHandleTypes); F(CUmemAllocationProp, location);
    F(CUmemAllocationProp, win32HandleMetaData); F(CUmemAllocationProp, allocFlags);
    F(CUmemAllocationProp, allocFlags.compressionType); F(CUmemAllocationProp, allocFlags.gpuDirectRDMACapable);
    F(CUmemAllocationProp, allocFlags.usage); F(CUmemAllocationProp, allocFlags.reserved);
    printf("CUmemAccessDesc - %zu %zu\n", sizeof(CUmemAccessDesc), _Alignof(CUmemAccessDesc));
    F(CUmemAccessDesc, location); F(CUmemAccessDesc, flags);
    return 0;
}
"""


def c_layout(tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(LAYOUT_PROBE)
    subprocess.check_call(["gcc", "-std=c11", "-I", cuda_include(), "-o", str(exe), str(src)])
    out = {}
    for line in subprocess.check_output([str(exe)], text=True).splitlines():
        name, field, a, b = line.split()
        out[(name, field)] = (int(a), int(b))
    return out


def field(struct, path):
    """(offset, size) of a dotted field of a ctypes struct."""
    off = 0
    for part in path.split("."):
        f = getattr(struct, part)
        off += f.offset
        typ = dict(struct._fields_)[part]
        struct = typ
    return off, f.size


def test_vmm_struct_layouts_match_cuda_h(tmp_path):
    want = c_layout(tmp_path)
    structs = {"CUmemLocation": sa.CUmemLocation, "CUmemAllocationProp": sa.CUmemAllocationProp,
               "CUmemAccessDesc": sa.CUmemAccessDesc}
    for (name, f), v in want.items():
        s = structs[name]
        got = (C.sizeof(s), C.alignment(s)) if f == "-" else field(s, f)
        assert got == v, (name, f, got, v)


def test_vmm_enums_match_cuda_h(tmp_path):
    src, exe = tmp_path / "enums.c", tmp_path / "enums"
    src.write_text("#include <cuda.h>\n#include <stdio.h>\nint main(void){printf(\"%d %d %d %d\\n\", (int)CU_MEM_ALLOCATION_TYPE_PINNED,"
                   "(int)CU_MEM_LOCATION_TYPE_DEVICE,(int)CU_MEM_ACCESS_FLAGS_PROT_READWRITE,(int)CU_MEM_ALLOC_GRANULARITY_MINIMUM);return 0;}\n")
    subprocess.check_call(["gcc", "-std=c11", "-I", cuda_include(), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [sa.CU_MEM_ALLOCATION_TYPE_PINNED, sa.CU_MEM_LOCATION_TYPE_DEVICE, sa.CU_MEM_ACCESS_FLAGS_PROT_READWRITE,
                   sa.CU_MEM_ALLOC_GRANULARITY_MINIMUM]


def test_a_moved_field_is_caught(tmp_path):
    """The layout check is not vacuous: a ctypes struct with two fields swapped differs from cuda.h."""
    want = c_layout(tmp_path)

    class Swapped(C.Structure):
        _fields_ = [("requestedHandleTypes", C.c_int), ("type", C.c_int), ("location", sa.CUmemLocation),
                    ("win32HandleMetaData", C.c_void_p), ("allocFlags", sa._AllocFlags)]
    assert field(Swapped, "type") != want[("CUmemAllocationProp", "type")]


# ---------------------------------------------------------------------------------------------------------------------
# mirror images
# ---------------------------------------------------------------------------------------------------------------------
def truncate(e, esz, how):
    """The address arithmetic a truncating caller does, written out with numpy's fixed-width integers."""
    if how == "u32_elem":
        return int(np.uint64(np.uint32(e & 0xFFFFFFFF))) * esz
    if how == "i32_elem":
        return int(np.int64(np.uint32(e & 0xFFFFFFFF).astype(np.int32))) * esz
    b = e * esz
    if how == "u32_byte":
        return int(np.uint32(b & 0xFFFFFFFF))
    return int(np.uint32(b & 0xFFFFFFFF).astype(np.int32))


OFFSET_CLASSES = [(1 << 30) + 4, (1 << 31) + 4, (1 << 31) - 8, (1 << 32) + 4, (1 << 32) - 12, (1 << 33) + 8, 3 << 31, 12]


@pytest.mark.parametrize("esz", [1, 2, 4, 8])
def test_images_cover_every_truncated_address(esz):
    rng = np.random.default_rng(esz)
    for lo in OFFSET_CLASSES:
        for n in (1, 4096, 3 << 20):
            ranges = sa.images(lo, n, esz)
            ranges.append((lo * esz, (lo + n) * esz))
            for e in [lo, lo + n - 1] + [int(v) for v in rng.integers(lo, lo + n, 64)] + \
                     [k for k in range(lo, lo + n, max(1, n // 16))]:
                for how in sa.TRUNCATIONS:
                    a = truncate(e, esz, how)
                    assert sa.image(e, esz, how) == a, (lo, n, e, how)
                    for byte in (a, a + esz - 1):
                        assert any(s <= byte < t for s, t in ranges), (lo, n, e, how, byte)
                    # every image lies inside the reservation: no lower than element 0 - base, no higher than 2^32 * esz
                    assert -sa.base_offset(esz) <= a < (1 << 32) * esz


def test_images_of_a_span_across_two_to_the_32():
    """A span that crosses 2^32 elements wraps under every 32-bit element truncation: its image is cut in two."""
    lo, n, esz = (1 << 32) - 256, 1024, 4
    ims = sa.images(lo, n, esz)
    u32 = sorted((a, b) for a, b in ims if a >= 0 and b <= (1 << 32) * esz)
    assert ((0, 768 * esz)) in u32 and (((1 << 32) - 256) * esz, (1 << 32) * esz) in u32


def test_runs_merge_and_clip():
    assert sa._runs([(5, 10), (8, 40), (100, 101), (-50, 3)], 16, 1 << 20) == [(0, 48), (96, 112)]
    assert sa._runs([(1 << 40, (1 << 40) + 1)], 16, 1 << 20) == []


# ---------------------------------------------------------------------------------------------------------------------
# copy-back planner past 2^32
# ---------------------------------------------------------------------------------------------------------------------
def cover(copies):
    """The element intervals a plan's copies write, merged."""
    iv = sorted((off + r * pitch, off + r * pitch + width) for off, width, pitch, height in copies for r in range(height))
    out = []
    for a, b in iv:
        assert not out or a >= out[-1][1], "two copies overlap"
        if out and a == out[-1][1]:
            out[-1] = (out[-1][0], b)
        else:
            out.append((a, b))
    return out


def want_cover(chans, chains, fmt):
    iv = []
    for C_, c in zip(chans, chains):
        if fmt == F32P:
            iv += [(c.out_offset + k * c.out_stride, c.out_offset + k * c.out_stride + c.n_samples) for k in range(C_) if c.n_samples]
        elif c.n_samples:
            iv.append((c.out_offset, c.out_offset + c.n_samples * C_))
    return cover([(a, b - a, 0, 1) for a, b in iv])


@pytest.mark.parametrize("shift", [(1 << 31) + 4, (1 << 32) + 4, (1 << 32) - 1000, (1 << 33) + 12, (1 << 40) + 8])
def test_copy_plan_translates_past_two_to_the_32(shift):
    """The plan of a layout moved by `shift` elements is the plan of the layout moved: same copies, offsets + shift."""
    S, Cn, stride = 16, 2, 3000
    for fmt in (F32P, F32I):
        small = [_Chain(s * Cn * stride, stride if fmt == F32P else 0, stride - 1024 * (s % 2)) for s in range(S)]
        big = [_Chain(c.out_offset + shift, c.out_stride, c.n_samples) for c in small]
        p_small, p_big = plan([Cn] * S, small, fmt), plan([Cn] * S, big, fmt)
        assert p_big == [(o + shift, w, p, h) for o, w, p, h in p_small]
        assert cover(p_big) == want_cover([Cn] * S, big, fmt)


@pytest.mark.parametrize("esz", [4, 2])
def test_copy_plan_with_pitches_past_two_to_the_32(esz):
    """Planar chains whose planes lie 2^32 + 4 elements apart: cut into rows at the library's pitch limit (INT32_MAX
    bytes), every plane copied once, at its 64-bit offset."""
    stride = (1 << 32) + 4
    chains = [_Chain((1 << 32) + 8, stride, 4000), _Chain((1 << 31) + 4, stride, 1500)]
    chans = [3, 2]
    for max_pitch in (1 << 40, (1 << 31) // esz - 1):
        p = plan(chans, chains, F32P, max_pitch)
        assert cover(p) == want_cover(chans, chains, F32P)
        assert all(h == 1 or pitch <= max_pitch for _, _, pitch, h in p)
        assert cover(p)[-1][1] == (1 << 32) + 8 + 2 * stride + 4000
