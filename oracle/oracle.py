"""ctypes binding of oracle/liblewton_oracle.so.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py -- never by lewton_b200/.
Every function is a thin wrapper; the arithmetic (and the reference file:line
citations) live in lewton_oracle.c.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liblewton_oracle.so")

MAX_POSTS = 65
FLOOR_UNUSED, FLOOR_ONE, FLOOR_DENSE = 0, 1, 2


def build(force=False):
    """Compile the oracle with gcc (oracle/Makefile)."""
    srcs = [os.path.join(_HERE, f) for f in ("lewton_oracle.c", "lwo_bench.c", "lewton_oracle.h",
                                             "floor1_inverse_db.inc", "Makefile")]
    if (not force and os.path.exists(_SO)
            and all(os.path.getmtime(_SO) >= os.path.getmtime(s) for s in srcs)):
        return _SO
    subprocess.check_call(["make", "-C", _HERE, "-B", "liblewton_oracle.so"],
                          stdout=subprocess.DEVNULL)
    return _SO


class Floor1(C.Structure):
    _fields_ = [("multiplier", C.c_int), ("nposts", C.c_int),
                ("x_list", C.c_uint32 * MAX_POSTS), ("sorted_idx", C.c_int * MAX_POSTS)]


class WindowGeom(C.Structure):
    _fields_ = [("n", C.c_int), ("left_start", C.c_int), ("left_end", C.c_int),
                ("right_start", C.c_int), ("right_end", C.c_int), ("left_use_bs1", C.c_int)]


class ChannelIn(C.Structure):
    _fields_ = [("floor_kind", C.c_int), ("fl", C.POINTER(Floor1)),
                ("floor1_y", C.POINTER(C.c_uint32)), ("dense_floor", C.POINTER(C.c_float)),
                ("residue", C.POINTER(C.c_float))]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        build()
    L = C.CDLL(_SO)
    vp, ip, fp = C.c_void_p, C.c_int, C.POINTER(C.c_float)
    L.lwo_tables_new.restype = vp
    L.lwo_tables_new.argtypes = [ip]
    L.lwo_tables_free.argtypes = [vp]
    for nm in ("a", "b", "c", "window"):
        f = getattr(L, "lwo_tables_" + nm)
        f.restype = fp
        f.argtypes = [vp]
    L.lwo_tables_bitrev.restype = C.POINTER(C.c_uint32)
    L.lwo_tables_bitrev.argtypes = [vp]
    L.lwo_inverse_mdct.argtypes = [vp, vp]
    L.lwo_inverse_mdct_slow.argtypes = [vp, ip]
    L.lwo_inverse_mdct_f64.argtypes = [vp, vp, ip]
    L.lwo_low_neighbor.argtypes = [vp, ip, C.POINTER(C.c_int), C.POINTER(C.c_uint32)]
    L.lwo_high_neighbor.argtypes = [vp, ip, C.POINTER(C.c_int), C.POINTER(C.c_uint32)]
    L.lwo_render_point.restype = C.c_uint32
    L.lwo_render_point.argtypes = [C.c_uint32] * 5
    L.lwo_floor1_sort.argtypes = [C.POINTER(Floor1)]
    L.lwo_floor1_amplitude.argtypes = [C.POINTER(Floor1), vp, vp, vp]
    L.lwo_floor1_synthesis.argtypes = [C.POINTER(Floor1), vp, vp, ip, vp]
    L.lwo_floor1_curve_y.argtypes = [C.POINTER(Floor1), vp, vp, ip, vp]
    L.lwo_inverse_db_table.restype = fp
    L.lwo_inverse_couple.argtypes = [vp, vp, ip]
    L.lwo_sample_i16.restype = C.c_int16
    L.lwo_sample_i16.argtypes = [C.c_float]
    L.lwo_window_geometry.argtypes = [ip] * 5 + [C.POINTER(WindowGeom)]
    L.lwo_pwr_new.restype = vp
    L.lwo_pwr_new.argtypes = [ip, ip]
    L.lwo_pwr_reset.argtypes = [vp]
    L.lwo_pwr_free.argtypes = [vp]
    L.lwo_pwr_has.argtypes = [vp]
    L.lwo_pwr_len.argtypes = [vp]
    L.lwo_pwr_data.restype = fp
    L.lwo_pwr_data.argtypes = [vp, ip]
    L.lwo_pwr_set.argtypes = [vp, ip]
    L.lwo_synth_packet.argtypes = [vp, vp, ip, ip, ip, ip, ip, vp, vp,
                                   C.POINTER(ChannelIn), vp, vp, C.POINTER(C.c_int)]
    L.lwo_synth_spectrum.argtypes = [vp, vp, ip, ip, ip, ip, vp, vp, vp, C.POINTER(C.c_int)]
    L.lwo_bench_chains.restype = C.c_double
    L.lwo_bench_chains.argtypes = [ip, ip, ip, vp, vp, ip, ip]
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class _TablesStruct(C.Structure):
    """lwo_tables (lewton_oracle.h), for tables held by numpy arrays."""
    _fields_ = [("bs", C.c_int), ("n", C.c_int), ("a", C.POINTER(C.c_float)), ("b", C.POINTER(C.c_float)),
                ("c", C.POINTER(C.c_float)), ("window", C.POINTER(C.c_float)), ("bitrev", C.POINTER(C.c_uint32))]


class Tables:
    """header_cached.rs:27-41 CachedBlocksizeDerived for one blocksize."""

    def __init__(self, bs):
        self.bs, self.n = bs, 1 << bs
        self._h = lib().lwo_tables_new(bs)
        self._owned = True
        if not self._h:
            raise ValueError("blocksize out of range")
        n = self.n
        L = lib()
        self.a = np.ctypeslib.as_array(L.lwo_tables_a(self._h), (n // 2,)).copy()
        self.b = np.ctypeslib.as_array(L.lwo_tables_b(self._h), (n // 2,)).copy()
        self.c = np.ctypeslib.as_array(L.lwo_tables_c(self._h), (n // 4,)).copy()
        self.window = np.ctypeslib.as_array(L.lwo_tables_window(self._h), (n // 2,)).copy()
        self.bitrev = np.ctypeslib.as_array(L.lwo_tables_bitrev(self._h), (n // 8,)).copy()

    @classmethod
    def from_arrays(cls, bs, a, b, c, window, bitrev):
        """Tables of the caller's own (a Rust caller's cached_bs_derived, or any other values): the oracle computes with
        exactly these arrays (copied; the attributes a, b, c, window and bitrev are read-only views of them, and the
        object keeps them alive for as long as the oracle reads them).  Not entered in the tables() cache."""
        if not 6 <= bs <= 13:
            raise ValueError("blocksize out of range")
        t = cls.__new__(cls)
        t.bs, t.n, t._owned = bs, 1 << bs, False
        n = t.n
        arrs = {}
        for name, arr, size, dt in (("a", a, n // 2, np.float32), ("b", b, n // 2, np.float32), ("c", c, n // 4, np.float32),
                                    ("window", window, n // 2, np.float32), ("bitrev", bitrev, n // 8, np.uint32)):
            x = np.array(arr, dt, copy=True).ravel()
            if x.size != size:
                raise ValueError(f"{name}: {size} entries expected for blocksize {bs}, got {x.size}")
            arrs[name] = x
            view = x.view()
            view.flags.writeable = False
            setattr(t, name, view)
        t._arrays = arrs                  # what _st points into, whatever becomes of the attributes
        t._st = _TablesStruct(bs, n, *(arrs[k].ctypes.data_as(C.POINTER(C.c_float)) for k in ("a", "b", "c", "window")),
                              arrs["bitrev"].ctypes.data_as(C.POINTER(C.c_uint32)))
        t._h = C.addressof(t._st)
        return t

    def __del__(self):
        try:
            if getattr(self, "_owned", False) and getattr(self, "_h", None) and _lib is not None:
                _lib.lwo_tables_free(self._h)
                self._h = None
        except Exception:
            pass


_tables = {}


def tables(bs):
    if bs not in _tables:
        _tables[bs] = Tables(bs)
    return _tables[bs]


def _pair(bs0, bs1, given):
    """The (blocksize_0, blocksize_1) tables: `given` (a pair of Tables) or the generated ones."""
    if given is None:
        return tables(bs0), tables(bs1)
    t0, t1 = given
    if (t0.bs, t1.bs) != (bs0, bs1):
        raise ValueError(f"tables of blocksizes {(t0.bs, t1.bs)} for a ({bs0}, {bs1}) stream")
    return t0, t1


def inverse_mdct(spectrum, bs, tables=None):
    """imdct.rs:291: n/2 coefficients -> n samples (float32).  tables: a Tables of blocksize bs (default: generated)."""
    t = _pair(bs, bs, None if tables is None else (tables, tables))[0]
    buf = np.zeros(t.n, np.float32)
    buf[: t.n // 2] = np.asarray(spectrum, np.float32)
    lib().lwo_inverse_mdct(t._h, _ptr(buf))
    return buf


def inverse_mdct_slow(spectrum, n):
    buf = np.zeros(n, np.float32)
    buf[: n // 2] = np.asarray(spectrum, np.float32)
    lib().lwo_inverse_mdct_slow(_ptr(buf), n)
    return buf


def inverse_mdct_f64(spectrum, n):
    s = np.ascontiguousarray(spectrum, np.float32)
    out = np.zeros(n, np.float64)
    lib().lwo_inverse_mdct_f64(_ptr(s), _ptr(out), n)
    return out


def low_neighbor(v, x):
    a = np.asarray(v, np.uint32)
    i, val = C.c_int(), C.c_uint32()
    if lib().lwo_low_neighbor(_ptr(a), x, C.byref(i), C.byref(val)):
        raise ValueError("no low neighbour (reference panics)")
    return i.value, val.value


def high_neighbor(v, x):
    a = np.asarray(v, np.uint32)
    i, val = C.c_int(), C.c_uint32()
    if lib().lwo_high_neighbor(_ptr(a), x, C.byref(i), C.byref(val)):
        raise ValueError("no high neighbour (reference panics)")
    return i.value, val.value


def render_point(x0, y0, x1, y1, x):
    return lib().lwo_render_point(x0, y0, x1, y1, x)


def make_floor1(multiplier, x_list):
    fl = Floor1()
    fl.multiplier = multiplier
    fl.nposts = len(x_list)
    for i, x in enumerate(x_list):
        fl.x_list[i] = x
    lib().lwo_floor1_sort(C.byref(fl))
    return fl


def floor1_amplitude(fl, floor1_y):
    y = np.asarray(floor1_y, np.uint32)
    fy = np.zeros(MAX_POSTS, np.uint32)
    s2 = np.zeros(MAX_POSTS, np.uint8)
    if lib().lwo_floor1_amplitude(C.byref(fl), _ptr(y), _ptr(fy), _ptr(s2)):
        raise ValueError("floor1 amplitude: reference would panic")
    return fy[: fl.nposts].copy(), s2[: fl.nposts].copy()


def floor1_curve_y(fl, final_y, step2, n2):
    fy = np.ascontiguousarray(final_y, np.uint32)
    s2 = np.ascontiguousarray(step2, np.uint8)
    out = np.zeros(n2, np.uint32)
    if lib().lwo_floor1_curve_y(C.byref(fl), _ptr(fy), _ptr(s2), n2, _ptr(out)):
        raise ValueError("floor1 curve: short")
    return out


def floor1_synthesis(fl, final_y, step2, n2):
    fy = np.ascontiguousarray(final_y, np.uint32)
    s2 = np.ascontiguousarray(step2, np.uint8)
    out = np.zeros(n2, np.float32)
    if lib().lwo_floor1_synthesis(C.byref(fl), _ptr(fy), _ptr(s2), n2, _ptr(out)):
        raise ValueError("floor1 synthesis: short")
    return out


def inverse_db_table():
    return np.ctypeslib.as_array(lib().lwo_inverse_db_table(), (256,)).copy()


def inverse_couple(mag, ang):
    m = np.array(mag, np.float32)
    a = np.array(ang, np.float32)
    lib().lwo_inverse_couple(_ptr(m), _ptr(a), len(m))
    return m, a


def sample_i16(x):
    x = np.asarray(x, np.float32)
    f = lib().lwo_sample_i16
    return np.array([f(float(v)) for v in x.ravel()], np.int16).reshape(x.shape)


def quantise_i16(x):
    """samples.rs:92-103, vectorised (bit-identical to sample_i16)."""
    x = np.asarray(x, np.float32)
    fl = x * np.float32(32768.0)
    out = np.where(np.isnan(fl), np.float32(0), fl)
    out = np.clip(np.trunc(out), -32768, 32767)
    return out.astype(np.int16)


def window_geometry(bs0, bs1, blockflag, prev_flag, next_flag):
    g = WindowGeom()
    lib().lwo_window_geometry(bs0, bs1, int(blockflag), int(prev_flag), int(next_flag), C.byref(g))
    return g


class Pwr:
    """audio.rs:847-861 PreviousWindowRight."""

    def __init__(self, channels, bs1):
        self.channels, self.cap = channels, (1 << bs1) // 2
        self._h = lib().lwo_pwr_new(channels, self.cap)

    def reset(self):
        lib().lwo_pwr_reset(self._h)

    def is_empty(self):
        return not lib().lwo_pwr_has(self._h)

    def __len__(self):
        return lib().lwo_pwr_len(self._h)

    def data(self):
        """[channels][len] copy, or None when empty."""
        if self.is_empty():
            return None
        n = len(self)
        return np.stack([np.ctypeslib.as_array(lib().lwo_pwr_data(self._h, c), (self.cap,))[:n].copy()
                         for c in range(self.channels)])

    def set_data(self, arr):
        arr = np.asarray(arr, np.float32)
        assert arr.shape[0] == self.channels and arr.shape[1] <= self.cap
        for c in range(self.channels):
            np.ctypeslib.as_array(lib().lwo_pwr_data(self._h, c), (self.cap,))[: arr.shape[1]] = arr[c]
        lib().lwo_pwr_set(self._h, arr.shape[1])

    def __del__(self):
        try:
            if getattr(self, "_h", None) and _lib is not None:
                _lib.lwo_pwr_free(self._h)
                self._h = None
        except Exception:
            pass


def synth_spectrum(bs0, bs1, blockflag, prev_flag, next_flag, spectrum, pwr, tables=None):
    """audio.rs:1041-1157 from the pre-MDCT tap.  spectrum [ch][n/2]; tables: (t0, t1) Tables (default: generated).
    Returns (rc, pcm[ch][len])."""
    t0, t1 = _pair(bs0, bs1, tables)
    n = (1 << bs1) if blockflag else (1 << bs0)
    sp = np.ascontiguousarray(spectrum, np.float32)
    ch = sp.shape[0]
    assert sp.shape[1] == n // 2
    out = np.zeros((ch, n), np.float32)
    olen = C.c_int(0)
    rc = lib().lwo_synth_spectrum(t0._h, t1._h, ch, int(blockflag), int(prev_flag), int(next_flag),
                                  _ptr(sp), pwr._h, _ptr(out), C.byref(olen))
    return rc, out[:, : olen.value].copy()


def synth_packet(bs0, bs1, blockflag, prev_flag, next_flag, coupling, floors, residues, pwr, tables=None):
    """audio.rs:988-1157.  coupling = [(mag, ang), ...] in header order;
    floors = per channel None | (Floor1, y[]) | ndarray(dense curve);
    residues [ch][n/2] (not modified); tables: (t0, t1) Tables (default: generated).  Returns (rc, pcm[ch][len])."""
    t0, t1 = _pair(bs0, bs1, tables)
    n = (1 << bs1) if blockflag else (1 << bs0)
    res = np.array(residues, np.float32, copy=True)
    ch = res.shape[0]
    assert res.shape[1] == n // 2
    chans = (ChannelIn * ch)()
    keep = []
    for c in range(ch):
        f = floors[c]
        chans[c].residue = res[c].ctypes.data_as(C.POINTER(C.c_float))
        if f is None:
            chans[c].floor_kind = FLOOR_UNUSED
        elif isinstance(f, np.ndarray):
            d = np.ascontiguousarray(f, np.float32)
            keep.append(d)
            chans[c].floor_kind = FLOOR_DENSE
            chans[c].dense_floor = d.ctypes.data_as(C.POINTER(C.c_float))
        else:
            fl, y = f
            ya = np.ascontiguousarray(y, np.uint32)
            keep.append(ya)
            chans[c].floor_kind = FLOOR_ONE
            chans[c].fl = C.pointer(fl)
            chans[c].floor1_y = ya.ctypes.data_as(C.POINTER(C.c_uint32))
    mag = np.array([m for m, _ in coupling], np.uint8)
    ang = np.array([a for _, a in coupling], np.uint8)
    out = np.zeros((ch, n), np.float32)
    olen = C.c_int(0)
    rc = lib().lwo_synth_packet(t0._h, t1._h, ch, int(blockflag), int(prev_flag), int(next_flag),
                                len(coupling), _ptr(mag), _ptr(ang), chans, pwr._h, _ptr(out),
                                C.byref(olen))
    return rc, out[:, : olen.value].copy()


def bench_chains(bs, spectrum, threads, reps=1):
    """spectrum [chains][packets][n/2] -> (seconds for `reps` passes, out [chains][(packets-1)*n/2 used])."""
    sp = np.ascontiguousarray(spectrum, np.float32)
    chains, packets, n2 = sp.shape
    out = np.zeros((chains, packets * n2), np.float32)
    sec = lib().lwo_bench_chains(bs, chains, packets, _ptr(sp), _ptr(out), threads, reps)
    return sec, out
