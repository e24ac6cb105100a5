"""Sparse arenas for batches at element offsets past 2^31 and 2^32, without the memory such offsets would take.

A device arena reserves a large virtual range with the CUDA driver's virtual memory management API (cuMemAddressReserve)
and maps physical memory only over windows: the spans a batch reads or writes and, for every such span, its images under
the four ways an address can be truncated to 32 bits (images()).  The arena's element 0 sits 2^31 elements, and at least
2 GiB, into the reservation, so that negative images are mapped as well.  Every window is filled with a sentinel, so a
32-bit truncation anywhere in the library shows up as a sentinel overwritten in a mirror window (or as a sentinel read
as data), not as a fault.  A host arena is an anonymous MAP_PRIVATE | MAP_NORESERVE mapping of which only the windows
are touched.  A host arena is the weaker check of the two: a stray write to an address that is neither a window nor one of
the four images lands in a fresh zero page that no check reads, where a device arena would fault.  The device cases are
the ones that pin the kernels down; the host cases pin down the host-side copies of a host-memory batch.

The ctypes layouts of the driver's structs are checked against cuda.h by tests/test_large_offsets_cpu.py."""
import ctypes as C
import mmap

import numpy as np

# ---------------------------------------------------------------------------------------------------------------------
# 32-bit images of an element span
# ---------------------------------------------------------------------------------------------------------------------
TRUNCATIONS = ("u32_elem", "i32_elem", "u32_byte", "i32_byte")
_M32, _H32 = 1 << 32, 1 << 31


def _trunc(v, signed):
    v %= _M32
    return v - _M32 if signed and v >= _H32 else v


def image(e, esz, how):
    """Byte offset from the arena's element 0 that element offset e reaches when the offset is truncated as `how`."""
    if how == "u32_elem":
        return _trunc(e, False) * esz
    if how == "i32_elem":
        return _trunc(e, True) * esz
    if how == "u32_byte":
        return _trunc(e * esz, False)
    if how == "i32_byte":
        return _trunc(e * esz, True)
    raise ValueError(how)


def images(lo, n, esz):
    """Byte ranges [a, b) relative to element 0 that cover the images of elements [lo, lo + n) under every truncation.
    Each image is linear between multiples of 2^31 elements and of 2^31 / esz elements; the span is cut there."""
    if n <= 0:
        return []
    cuts = {lo, lo + n}
    for unit in (_H32, _H32 // esz):
        k = (lo // unit + 1) * unit
        while k < lo + n:
            cuts.add(k)
            k += unit
    cuts = sorted(cuts)
    out = []
    for a, b in zip(cuts, cuts[1:]):
        for how in TRUNCATIONS:
            s = image(a, esz, how)
            out.append((s, s + (b - a) * esz))
    return out


def base_offset(esz):
    """Bytes from a reservation's start to the arena's element 0: 2^31 elements, and at least 2 GiB."""
    return max(_H32 * esz, _H32)


# ---------------------------------------------------------------------------------------------------------------------
# CUDA driver VMM, through ctypes
# ---------------------------------------------------------------------------------------------------------------------
class CUmemLocation(C.Structure):
    _fields_ = [("type", C.c_int), ("id", C.c_int)]


class _AllocFlags(C.Structure):
    _fields_ = [("compressionType", C.c_ubyte), ("gpuDirectRDMACapable", C.c_ubyte), ("usage", C.c_ushort),
                ("reserved", C.c_ubyte * 4)]


class CUmemAllocationProp(C.Structure):
    _fields_ = [("type", C.c_int), ("requestedHandleTypes", C.c_int), ("location", CUmemLocation),
                ("win32HandleMetaData", C.c_void_p), ("allocFlags", _AllocFlags)]


class CUmemAccessDesc(C.Structure):
    _fields_ = [("location", CUmemLocation), ("flags", C.c_int)]


CU_MEM_ALLOCATION_TYPE_PINNED = 1
CU_MEM_LOCATION_TYPE_DEVICE = 1
CU_MEM_ACCESS_FLAGS_PROT_READWRITE = 3
CU_MEM_ALLOC_GRANULARITY_MINIMUM = 0

_cuda = None


def driver():
    global _cuda
    if _cuda is None:
        lib = C.CDLL("libcuda.so.1")
        u64, p = C.c_uint64, C.POINTER
        lib.cuMemAddressReserve.argtypes = [p(u64), C.c_size_t, C.c_size_t, u64, u64]
        lib.cuMemAddressFree.argtypes = [u64, C.c_size_t]
        lib.cuMemCreate.argtypes = [p(u64), C.c_size_t, p(CUmemAllocationProp), u64]
        lib.cuMemRelease.argtypes = [u64]
        lib.cuMemMap.argtypes = [u64, C.c_size_t, C.c_size_t, u64, u64]
        lib.cuMemUnmap.argtypes = [u64, C.c_size_t]
        lib.cuMemSetAccess.argtypes = [u64, C.c_size_t, p(CUmemAccessDesc), C.c_size_t]
        lib.cuMemGetAllocationGranularity.argtypes = [p(C.c_size_t), p(CUmemAllocationProp), C.c_int]
        _cuda = lib
    return _cuda


def _ck(rc, what):
    if rc:
        raise RuntimeError(f"{what}: CUresult {rc}")


def _runs(ranges, gran, limit):
    """Granule-aligned, merged runs [a, b) covering the byte ranges, clipped to [0, limit)."""
    gs = []
    for a, b in ranges:
        a, b = max(0, a // gran * gran), min(limit, -(-b // gran) * gran)
        if a < b:
            gs.append((a, b))
    gs.sort()
    out = []
    for a, b in gs:
        if out and a <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], b))
        else:
            out.append((a, b))
    return out


_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}     # the sentinel's word, by element size


class _Sparse:
    """What the device and host arenas share: element spans to cover, their mirror images, and the windows mapped."""

    def __init__(self, dtype, guard, max_elems):
        self.dtype, self.guard = np.dtype(dtype), guard
        self.esz = self.dtype.itemsize
        self.base = base_offset(self.esz)
        self.size = self.base + max(max_elems * self.esz, _M32 * self.esz) + (64 << 20)
        self.spans, self.ranges, self.windows = [], [], []

    def cover(self, lo, n):
        """Element span [lo, lo + n) of the batch, and its 32-bit images."""
        assert lo >= 0 and (lo + n) * self.esz + self.base <= self.size
        self.spans.append((lo, n))
        self.ranges.append((self.base + lo * self.esz, self.base + (lo + n) * self.esz))
        self.ranges += [(self.base + a, self.base + b) for a, b in images(lo, n, self.esz)]

    def mapped(self, byte_off):
        """Whether byte `byte_off` from element 0 lies in a mapped window."""
        b = self.base + byte_off
        return any(a <= b < e for a, e in self.windows)

    def _guard_words(self, nbytes):
        u = _UINT[self.esz]
        return np.full(nbytes // self.esz, self.guard, u)

    def bits(self, a):
        return a.view(_UINT[self.esz])

    def check_guard(self, write_spans, what):
        """Every element of every window outside `write_spans` [(lo, n)] still holds the sentinel."""
        for a, b in self.windows:
            got = self.bits(self.read_bytes(a, b - a))
            keep = np.ones(got.size, bool)
            e0 = (a - self.base) // self.esz
            for lo, n in write_spans:
                s, t = max(lo - e0, 0), min(lo + n - e0, got.size)
                if s < t:
                    keep[s:t] = False
            bad = np.nonzero(keep & (got != self.guard))[0]
            if bad.size:
                e = e0 + int(bad[0])
                real = any(lo <= e < lo + n for lo, n in self.spans)
                raise AssertionError(f"{what}: {bad.size} sentinels overwritten in the {'batch' if real else 'mirror'} "
                                     f"window at element {e0} ({(b - a) // self.esz} elements); first at element {e}")


class DeviceArena(_Sparse):
    """A sparse device arena of `dtype`, element 0 at .ptr; windows mapped over cover()ed spans by commit()."""

    def __init__(self, dtype, guard, max_elems, device=0):
        super().__init__(dtype, guard, max_elems)
        self.device = device
        drv = driver()
        self.prop = CUmemAllocationProp()
        self.prop.type = CU_MEM_ALLOCATION_TYPE_PINNED
        self.prop.location.type, self.prop.location.id = CU_MEM_LOCATION_TYPE_DEVICE, device
        g = C.c_size_t()
        _ck(drv.cuMemGetAllocationGranularity(C.byref(g), C.byref(self.prop), CU_MEM_ALLOC_GRANULARITY_MINIMUM), "granularity")
        self.gran = g.value
        self.size = -(-self.size // self.gran) * self.gran
        r = C.c_uint64()
        _ck(drv.cuMemAddressReserve(C.byref(r), self.size, 0, 0, 0), "cuMemAddressReserve")
        self.res = r.value
        self.ptr = self.res + self.base
        self.handles = []

    def commit(self, ctx):
        """Maps every window and fills it with the sentinel (ctx: the lewton_b200 Context whose stream copies)."""
        drv = driver()
        acc = CUmemAccessDesc()
        acc.location.type, acc.location.id = CU_MEM_LOCATION_TYPE_DEVICE, self.device
        acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE
        for a, b in _runs(self.ranges, self.gran, self.size):
            h = C.c_uint64()
            _ck(drv.cuMemCreate(C.byref(h), b - a, C.byref(self.prop), 0), "cuMemCreate")
            self.handles.append((h.value, None))
            _ck(drv.cuMemMap(self.res + a, b - a, 0, h.value, 0), "cuMemMap")
            self.handles[-1] = (h.value, (a, b))
            _ck(drv.cuMemSetAccess(self.res + a, b - a, C.byref(acc), 1), "cuMemSetAccess")
            self.windows.append((a, b))
            ctx.h2d(self.res + a, self._guard_words(b - a))
        self.ctx = ctx
        return self

    def physical_bytes(self):
        return sum(b - a for a, b in self.windows)

    def write(self, lo, arr):
        self.ctx.h2d(self.ptr + lo * self.esz, np.ascontiguousarray(arr, self.dtype))

    def read(self, lo, n):
        out = np.empty(n, self.dtype)
        self.ctx.d2h(out, self.ptr + lo * self.esz)
        return out

    def read_bytes(self, a, nbytes):
        out = np.empty(nbytes // self.esz, self.dtype)
        self.ctx.d2h(out, self.res + a)
        return out

    def close(self):
        """After the context has synchronised: unmaps and frees every window, then the reservation."""
        drv = driver()
        for h, ab in self.handles:
            if ab:
                drv.cuMemUnmap(self.res + ab[0], ab[1] - ab[0])
            drv.cuMemRelease(h)
        self.handles, self.windows = [], []
        if self.res:
            drv.cuMemAddressFree(self.res, self.size)
            self.res = 0


# Linux's MAP_NORESERVE (Python's mmap module does not name it)
MAP_NORESERVE = 0x4000


class HostArena(_Sparse):
    """A sparse host arena: an anonymous private mapping that reserves no swap; only the windows are touched.  .arr is the
    whole mapping as a numpy array from element 0 on (the address a batch's io takes); .page_lock() registers one span."""

    def __init__(self, dtype, guard, max_elems):
        super().__init__(dtype, guard, max_elems)
        self.gran = mmap.PAGESIZE
        self.size = -(-self.size // self.gran) * self.gran
        self.mm = mmap.mmap(-1, self.size, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | MAP_NORESERVE)
        self.whole = np.frombuffer(self.mm, np.uint8)
        self.arr = self.whole[self.base:].view(self.dtype)
        self.registered = []

    def commit(self, ctx=None):
        for a, b in _runs(self.ranges, self.gran, self.size):
            self.whole[a:b].view(self._guard_words(0).dtype)[...] = self.guard
            self.windows.append((a, b))
        return self

    def physical_bytes(self):
        return sum(b - a for a, b in self.windows)

    def write(self, lo, arr):
        self.arr[lo:lo + len(arr)] = np.asarray(arr, self.dtype)

    def read(self, lo, n):
        return self.arr[lo:lo + n].copy()

    def read_bytes(self, a, nbytes):
        return self.whole[a:a + nbytes].view(self.dtype).copy()

    def page_lock(self, lo, n):
        """cudaHostRegister over the pages of elements [lo, lo + n) (a host-memory submit's extent)."""
        import torch
        a = (self.base + lo * self.esz) // self.gran * self.gran
        b = -(-(self.base + (lo + n) * self.esz) // self.gran) * self.gran
        addr = self.whole[a:].ctypes.data
        torch.cuda.check_error(torch.cuda.cudart().cudaHostRegister(addr, b - a, 0))
        self.registered.append(addr)

    def close(self):
        """After the context has synchronised: unregisters the page-locked spans and drops the mapping."""
        import torch
        for addr in self.registered:
            torch.cuda.check_error(torch.cuda.cudart().cudaHostUnregister(addr))
        self.registered = []
        self.arr = self.whole = None
        try:
            self.mm.close()
        except BufferError:
            # numpy views of the mapping that a test still holds (the arrays a marshalled io pointed to, kept alive by a
            # traceback) pin it; the mapping then goes with the last of them.  It reserves no swap, and only its windows
            # were ever touched.
            pass
