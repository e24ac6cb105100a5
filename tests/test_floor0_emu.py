"""CPU emulation of the GPU's floor-0 curve synthesis (tests/emu/floor0_emu.cpp compiles
lewton_b200/csrc/kernel_floor0.cuh for the host): the restated expf and the FMA-free division and square root against
the host's libm on every input, and the per-bin row renderer against floor0_expected (the reference's run walk of
audio.rs:160-212 in f32, libm through ctypes) on random floors and edge cases."""
import ctypes as C
import os
import platform
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import numpy as np
import pytest

from test_frontend_cpu import floor0_expected, libm

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "emu", "liblwb_floor0_emu.so")


def build():
    src = os.path.join(HERE, "emu", "floor0_emu.cpp")
    deps = [src] + [os.path.join(HERE, "..", "lewton_b200", "csrc", f) for f in ("kernel_floor0.cuh", "lwb_common.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-I",
                               os.path.join(HERE, "..", "include"), "-o", SO, src, "-lm"])
    return SO


def emu():
    L = C.CDLL(build())
    L.lwb_emu_unary_mismatches.restype = C.c_uint64
    L.lwb_emu_unary_mismatches.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
    L.lwb_emu_div_mismatches.restype = C.c_uint64
    L.lwb_emu_div_mismatches.argtypes = [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
    L.lwb_emu_floor0_row.restype = None
    L.lwb_emu_floor0_row.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return L


def _all_inputs(op):
    """(mismatches, first mismatching input) of unary op over all 2^32 float bit patterns, on every core."""
    L = emu()
    parts = max(1, min(64, os.cpu_count() or 1) * 4)
    step = (1 << 32) // parts

    def run(i):
        first = C.c_uint32(0)
        lo = i * step
        hi = (1 << 32) if i == parts - 1 else lo + step
        return L.lwb_emu_unary_mismatches(op, lo, hi, C.byref(first)), first.value

    with ThreadPoolExecutor(parts) as ex:           # ctypes releases the GIL for the call
        res = list(ex.map(run, range(parts)))
    bad = [(n, f) for n, f in res if n]
    return sum(n for n, _ in res), (bad[0][1] if bad else None)


def _libc():
    return platform.libc_ver()


def test_restated_expf_equals_the_hosts_expf_on_every_input():
    """d_expf is glibc's expf (>= 2.28) restated without FMA; the reference calls the platform expf.  If this host's libm
    computes expf differently, the failure says so: the device then matches glibc, not this host."""
    n, first = _all_inputs(0)
    assert n == 0, (f"{n} inputs where the restated expf differs from this host's expf ({_libc()}); first: "
                    f"{np.uint32(first).view(np.float32).item().hex()} (bits 0x{first:08x})")


def test_fma_free_sqrt_equals_sqrtf_on_every_input():
    n, first = _all_inputs(1)
    assert n == 0, f"{n} mismatches, first bits 0x{first:08x}"


def test_fma_free_division_equals_ieee_division():
    L = emu()
    first = (C.c_uint32 * 2)()
    with ThreadPoolExecutor(8) as ex:
        res = list(ex.map(lambda s: (L.lwb_emu_div_mismatches(s, 20_000_000, first), tuple(first)), range(1, 9)))
    assert sum(n for n, _ in res) == 0, [f"0x{a:08x}/0x{b:08x}" for n, (a, b) in res if n]


# ---- records and tables, as the host front half produces them -------------------------------------------------------
def bark_cos_omega(rate, bark_map_size, n):
    """cached_bark_cos_omega (header_cached.rs:129-158) in f32 with libm, as floor0_expected computes it."""
    m = libm()
    atanf = C.CDLL("libm.so.6").atanf
    atanf.argtypes, atanf.restype = [C.c_float], C.c_float
    f32 = np.float32

    def bark(x):
        x = f32(x)
        return f32(f32(f32(13.1) * f32(atanf(f32(f32(0.00074) * x)))) + f32(f32(2.24) * f32(atanf(f32(f32(f32(0.0000000185) * x) * x))))) + f32(f32(0.0001) * x)

    hfl = f32(f32(rate) / f32(2.0))
    hfl_dn = f32(hfl / f32(n))
    const = f32(f32(bark_map_size) / f32(bark(hfl)))
    bms_m1 = f32(f32(bark_map_size) - f32(1.0))
    omega_factor = f32(f32(np.pi) / f32(bark_map_size))
    out = np.zeros(n, f32)
    for i in range(n):
        fb = f32(np.floor(f32(f32(bark(f32(f32(i) * hfl_dn))) * const)))
        out[i] = f32(m.cosf(f32(min(fb, bms_m1) * omega_factor)))
    return out


def coeff_cosines(order, rows):
    """floor_zero_decode's coefficients (audio.rs:131-145): cosf(last + e) over the VQ rows."""
    m = libm()
    f32 = np.float32
    coeffs, last = [], f32(0)
    for row in rows:
        last_new = last
        for e in row:
            coeffs.append(f32(m.cosf(f32(last + f32(e)))))
            last_new = f32(e)
            if len(coeffs) == order:
                break
        last = f32(last + last_new)
        if len(coeffs) >= order:
            break
    return np.array(coeffs, f32)


def record_words(amp, cosc):
    """The LWB_FLOOR_ZERO record of a row: amplitude (u64, low word first) then the cosines' bits, in LWB_MAX_POSTS words."""
    w = np.zeros(65, np.uint32)
    w[0], w[1] = amp & 0xffffffff, amp >> 32
    w[2: 2 + len(cosc)] = np.asarray(cosc, np.float32).view(np.uint32)
    return w


def render(L, fl, amp, cosc, bark):
    out = np.zeros(len(bark), np.float32)
    cosc = np.ascontiguousarray(cosc, np.float32)
    bark = np.ascontiguousarray(bark, np.float32)
    L.lwb_emu_floor0_row(fl.order, fl.amplitude_bits, fl.amplitude_offset, amp, cosc.ctypes.data, bark.ctypes.data, len(bark),
                         out.ctypes.data)
    return out


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | nan))


def random_amplitude(rng, bits):
    """A nonzero amplitude of `bits` bits with at most 53 significant bits (numpy's f32 of a Python int goes through
    double) -- or the all-ones maximum."""
    if rng.random() < 0.2:
        return (1 << bits) - 1
    if bits <= 53:
        return int(rng.integers(1, 1 << bits, dtype=np.uint64)) if bits < 64 else 1
    return int(rng.integers(1, 1 << 53, dtype=np.uint64)) << (bits - 53)


@pytest.mark.parametrize("seed", range(6))
def test_row_renderer_matches_floor0_expected_on_random_floors(seed):
    L = emu()
    rng = np.random.default_rng(4000 + seed)
    pairs = [(b0, b1) for b0 in range(6, 14) for b1 in range(b0, 14)]
    for case in range(10):
        bs0, bs1 = pairs[(seed * 10 + case) % len(pairs)]
        order = int(rng.integers(2, 64))
        bits = int(rng.integers(1, 65))
        fl = SimpleNamespace(order=order, amplitude_bits=bits, amplitude_offset=int(rng.integers(0, 256)),
                             rate=int(rng.choice([8, 1000, 8000, 22050, 44100, 65535])), bark_map_size=int(rng.choice([1, 7, 64, 256, 4000, 65535])))
        amp = random_amplitude(rng, bits)
        dim = int(rng.integers(1, 9))
        rows = [list(rng.uniform(-0.5, 3.5, dim).astype(np.float32)) for _ in range((order + dim - 1) // dim)]
        cosc = coeff_cosines(order, rows)
        for blockflag in (0, 1):
            n2 = 1 << ((bs1 if blockflag else bs0) - 1)
            if n2 > 512 and case % 3:                 # (the Python oracle is slow: every third case at the large sizes)
                continue
            bark = bark_cos_omega(fl.rate, fl.bark_map_size, n2)
            want = floor0_expected(fl, amp, rows, blockflag, n2, bs0, bs1)
            got = render(L, fl, amp, cosc, bark)
            assert same_bits(got, want), (seed, case, blockflag, np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0][:5])


def _expected_from_table(fl, amp, cosc, bark):
    """floor0_expected's run walk over a given bark table (synthetic tables reach the edge cases)."""
    m = libm()
    f32 = np.float32
    common = f32(f32(f32(amp) * f32(fl.amplitude_offset)) / f32((1 << fl.amplitude_bits) - 1))
    out = np.zeros(len(bark), f32)
    i = 0
    with np.errstate(all="ignore"):
        while i < len(bark):
            co = bark[i]
            if fl.order & 1:
                pu, qu = (fl.order - 3) // 2, (fl.order - 1) // 2
                p, q = f32(f32(1.0) - f32(co * co)), f32(0.25)
            else:
                pu = qu = (fl.order - 2) // 2
                p, q = f32(f32(f32(1.0) - co) / f32(2.0)), f32(f32(f32(1.0) + co) / f32(2.0))
            for j in range(pu + 1):
                pm = f32(cosc[2 * j + 1] - co)
                p = f32(p * f32(f32(f32(4.0) * pm) * pm))
            for j in range(qu + 1):
                qm = f32(cosc[2 * j] - co)
                q = f32(q * f32(f32(f32(4.0) * qm) * qm))
            lfv = f32(m.expf(f32(f32(0.11512925) * f32(f32(common / f32(m.sqrtf(f32(p + q)))) - f32(fl.amplitude_offset)))))
            while i < len(bark) and bark[i] == co:
                out[i] = lfv
                i += 1
    return out


def test_row_renderer_edge_cases():
    """p + q == 0 (common / 0: inf, or NaN with a zero offset), negative p + q (a caller's table beyond [-1, 1]: NaN),
    exp overflowing to inf, a coefficient equal to cos_omega, long runs of equal cos_omega.  (Subnormal curve values
    need an exp argument below -87, which 0.11512925 * (common / sqrt(p + q) - offset) >= -29.4 never reaches; d_expf's
    subnormal outputs are covered by the all-inputs test.)"""
    L = emu()
    f32 = np.float32
    runs = np.repeat(np.array([1.0, 0.75, 0.75, -0.25, -1.0], f32), [3, 40, 1, 100, 4])
    cases = [
        (SimpleNamespace(order=2, amplitude_bits=8, amplitude_offset=100), 200, np.array([1.0, 0.5], f32), runs),      # p + q == 0 at bin 0
        (SimpleNamespace(order=2, amplitude_bits=8, amplitude_offset=0), 200, np.array([1.0, 0.5], f32), runs),        # 0 / 0
        (SimpleNamespace(order=3, amplitude_bits=4, amplitude_offset=50), 9, np.array([0.1, 0.2, 0.3], f32),
         np.array([3.0, 1.5, -3.0, 0.5], f32)),                                                                       # p + q < 0
        (SimpleNamespace(order=4, amplitude_bits=64, amplitude_offset=255), (1 << 64) - 1, np.array([0.75, 0.75, 0.75, 0.75], f32),
         np.array([0.75, 0.7500001, 0.74999994, 0.75], f32)),                                                       # overflow to inf
        (SimpleNamespace(order=5, amplitude_bits=12, amplitude_offset=7), 1234, np.array([-0.25, 0.75, 0.3, -1.0, 0.9], f32), runs),
    ]
    for k, (fl, amp, cosc, bark) in enumerate(cases):
        want = _expected_from_table(fl, amp, cosc, bark)
        got = render(L, fl, amp, cosc, bark)
        assert same_bits(got, want), (k, got[:8], want[:8])
    assert np.isinf(render(L, *cases[0][:3], cases[0][3])[0]) and np.isnan(render(L, *cases[1][:3], cases[1][3])[0])
    assert np.isnan(render(L, *cases[2][:3], cases[2][3])[0]) and np.isinf(render(L, *cases[3][:3], cases[3][3])).any()
