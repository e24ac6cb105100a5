// kernel_floor0.cuh -- floor type 0 curve synthesis (floor_zero_compute_curve, audio.rs:160-212) on the device, bit for
// bit.  The row math is host+device (LWB_HD) so that tests/emu/floor0_emu.cpp runs exactly this source on the CPU.
//
// What the device gets per (packet, channel) row of kind LWB_FLOOR_ZERO: the packet's floor-0 record in the row's
// floor1_y words (amplitude as a u64, low word first, then the `order` coefficient cosines as f32 bit patterns --
// floor_zero_decode's output, audio.rs:131-145, whose cosf stays on the host), and per setup the floor's constants and
// its cached_bark_cos_omega tables (header_cached.rs:129-158, also libm on the host).  What is left is f32 multiply and
// add, a division and a square root (d_fdiv / d_fsqrt: IEEE-exact without FMA) and one expf, which d_expf restates
// exactly.
#pragma once
#include <stdint.h>
#include <string.h>

#include "kernel_long.cuh"      // LWB_HD
#include "lwb_common.h"

namespace lwb {

// ---------------------------------------------------------------------------------------------
// glibc's expf (sysdeps/ieee754/flt-32/e_expf.c, glibc >= 2.28), restated in double arithmetic so that it gives the
// same float for every input.  exp(x) = 2^(k/32) * 2^(r/32) with x * 32/ln2 = k + r: a 32-entry table of 2^(i/32)
// and a cubic polynomial in r, rounded to float once at the end.  The x86-64 build of glibc that the reference links
// (its FMA variant) rounds the reduction r = x * 32/ln2 - k once; without a fused multiply-add (the project's SASS has
// none, see build.check_no_fma) that single rounding comes from an exact split of 32/ln2 = kInvLn2NHi + kInvLn2NLo:
// x * kInvLn2NHi (24 x 25 bits) and x * kInvLn2NLo (24 x 26 bits) are exact, and so is x * kInvLn2NHi - k, so
// (x * kInvLn2NHi - k) + x * kInvLn2NLo rounds once.  The polynomial is evaluated unfused.
// ---------------------------------------------------------------------------------------------
LWB_HD double d0_mul(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
LWB_HD double d0_add(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
LWB_HD double d0_bits_to_double(uint64_t u)
{
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double d;
    memcpy(&d, &u, sizeof(d));
    return d;
#endif
}
LWB_HD uint64_t d0_double_to_bits(double d)
{
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u;
    memcpy(&u, &d, sizeof(u));
    return u;
#endif
}
LWB_HD uint32_t d0_float_to_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, sizeof(u));
    return u;
#endif
}
LWB_HD float d0_bits_to_float(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, sizeof(f));
    return f;
#endif
}

// bits(2^(i/32)) - (i << 47): adding k << 47 back puts k / 32 into the exponent.  One table for the host, one in
// constant memory for the device.
#define LWB_EXP_TAB {                                                                   \
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, \
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, \
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull, \
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, \
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull, \
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull, \
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, \
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull }
static const uint64_t h_exp_tab[32] = LWB_EXP_TAB;
#if defined(__CUDACC__)
__constant__ uint64_t c_exp_tab[32] = LWB_EXP_TAB;
#endif
#undef LWB_EXP_TAB

LWB_HD float d_expf(float x)
{
    const uint32_t ux = d0_float_to_bits(x);
    if ((ux & 0x7fffffffu) > 0x7f800000u) return x + x;          // NaN
    if (x > 0x1.62e42ep6f) return d0_bits_to_float(0x7f800000u);    // x > log(0x1p128): +inf
    if (x < -0x1.9fe368p6f) return 0.0f;                          // x < log(0x1p-150): +0 (and -inf)
    const double kInvLn2N = 0x1.71547652b82fep+5;                 // 32 / ln2
    const double kInvLn2NHi = 0x1.715476p+5, kInvLn2NLo = 0x1.4ae0bf8p-21;
    const double kShift = 0x1.8p52;
    const double xd = (double)x;
    double kd = d0_add(d0_mul(kInvLn2N, xd), kShift);             // round to an integer, ties to even
    const uint64_t ki = d0_double_to_bits(kd);
    kd = d0_add(kd, -kShift);
    const double r = d0_add(d0_add(d0_mul(xd, kInvLn2NHi), -kd), d0_mul(xd, kInvLn2NLo));
#if defined(__CUDA_ARCH__)
    const double s = d0_bits_to_double(c_exp_tab[ki % 32] + (ki << 47));
#else
    const double s = d0_bits_to_double(h_exp_tab[ki % 32] + (ki << 47));
#endif
    const double z = d0_add(d0_mul(0x1.c6af84b912394p-20, r), 0x1.ebfce50fac4f3p-13);
    const double r2 = d0_mul(r, r);
    double y = d0_add(d0_mul(0x1.62e42ff0c52d6p-6, r), 1.0);
    y = d0_add(d0_mul(z, r2), y);
    y = d0_mul(y, s);
#if defined(__CUDA_ARCH__)
    return __double2float_rn(y);
#else
    return (float)y;
#endif
}

// ---------------------------------------------------------------------------------------------
// IEEE f32 division and square root, correctly rounded, without a fused multiply-add.  The device's own div.rn / sqrt.rn
// refine their estimates with FFMA; these take a double estimate (Newton iterations in double multiply and add) and
// settle the rounding exactly: the result is the float f whose two rounding midpoints m- < m+ (25-bit numbers) bracket
// the exact value, and b * m (for a / b) or m * m (for sqrt) is exact in double, so the comparisons are exact.
// ---------------------------------------------------------------------------------------------
LWB_HD double d0_value_of_bits(uint32_t u)                      // value of a non-negative bit pattern; 0x7f800000 = 2^128
{
    return u >= 0x7f800000u ? 0x1p128 : (double)d0_bits_to_float(u);
}
// u: bits of a non-negative finite or infinite float approximating x = num / den (den > 0, both exact in double, den *
// midpoint exact); returns the bits of the correctly rounded x.  Exact midpoints (possible in the subnormal range) round
// to even.
LWB_HD uint32_t d0_settle(uint32_t u, double num, double den)
{
    const double mid = d0_value_of_bits(u);
    if (u > 0) {
        const double lo = d0_value_of_bits(u - 1);
        const double m = d0_mul(den, d0_mul(d0_add(lo, mid), 0.5));
        if (num < m || (num == m && (u & 1))) return u - 1;
    }
    if (u < 0x7f800000u) {
        const double hi = d0_value_of_bits(u + 1);
        const double m = d0_mul(den, d0_mul(d0_add(mid, hi), 0.5));
        if (num > m || (num == m && (u & 1))) return u + 1;
    }
    return u;
}
LWB_HD uint32_t d0_double_to_float_bits(double d)
{
#if defined(__CUDA_ARCH__)
    return d0_float_to_bits(__double2float_rn(d));
#else
    return d0_float_to_bits((float)d);
#endif
}

LWB_HD float d_fdiv(float a, float b)
{
    const uint32_t ua = d0_float_to_bits(a), ub = d0_float_to_bits(b);
    const uint32_t sign = (ua ^ ub) & 0x80000000u, aa = ua & 0x7fffffffu, ab = ub & 0x7fffffffu;
    if (aa > 0x7f800000u || ab > 0x7f800000u) return a + b;                            // NaN
    if ((aa == 0 && ab == 0) || (aa == 0x7f800000u && ab == 0x7f800000u)) return d0_bits_to_float(0x7fc00000u);
    if (aa == 0x7f800000u || ab == 0) return d0_bits_to_float(sign | 0x7f800000u);   // inf
    if (aa == 0 || ab == 0x7f800000u) return d0_bits_to_float(sign);                 // 0
    const double A = (double)d0_bits_to_float(aa), B = (double)d0_bits_to_float(ab);
    double y = d0_bits_to_double(0x7fde623822fc16e6ull - d0_double_to_bits(B));     // 1/B to ~12 %
    for (int i = 0; i < 5; i++) y = d0_mul(y, d0_add(2.0, -d0_mul(B, y)));           // error squared per step
    const uint32_t u = d0_settle(d0_double_to_float_bits(d0_mul(A, y)), A, B);
    return d0_bits_to_float(sign | u);
}

LWB_HD float d_fsqrt(float x)
{
    const uint32_t ux = d0_float_to_bits(x);
    if ((ux & 0x7fffffffu) == 0 || ux == 0x7f800000u) return x;                     // +-0, +inf
    if (ux > 0x7f800000u) return (ux & 0x7fffffffu) > 0x7f800000u ? x + x : d0_bits_to_float(0xffc00000u);   // NaN, x < 0
    const double X = (double)x;
    double y = d0_bits_to_double(0x5fe6eb50c7b537a9ull - (d0_double_to_bits(X) >> 1));   // 1/sqrt(X) to ~3.5 %
    for (int i = 0; i < 4; i++) y = d0_mul(y, d0_add(1.5, -d0_mul(d0_mul(0.5, X), d0_mul(y, y))));
    const uint32_t u = d0_double_to_float_bits(d0_mul(X, y));
    // sqrt: the midpoints are compared through their squares, X against m * m
    const double lo = d0_value_of_bits(u - 1), mid = d0_value_of_bits(u), hi = d0_value_of_bits(u + 1);
    const double ml = d0_mul(d0_add(lo, mid), 0.5), mh = d0_mul(d0_add(mid, hi), 0.5);
    if (X < d0_mul(ml, ml)) return d0_bits_to_float(u - 1);
    if (X > d0_mul(mh, mh)) return d0_bits_to_float(u + 1);
    return d0_bits_to_float(u);
}

// ---------------------------------------------------------------------------------------------
// one bin of floor_zero_compute_curve, audio.rs:160-212, in its f32 rounding order
// ---------------------------------------------------------------------------------------------
LWB_HD float f0_mul(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
LWB_HD float f0_add(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
LWB_HD float f0_sub(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}

// max_amp of audio.rs:167-169 as f32; 64 amplitude bits are legal (header.rs:780-787) and give u64::MAX
LWB_HD float d_floor0_max_amp(int amplitude_bits)
{
    return (float)(amplitude_bits >= 64 ? ~0ull : ((1ull << amplitude_bits) - 1));
}

// common = amplitude * amplitude_offset / max_amp (audio.rs:167-169), once per row
LWB_HD float d_floor0_common(uint64_t amplitude, uint32_t amplitude_offset, float max_amp)
{
#if defined(__CUDA_ARCH__)
    const float a = __ull2float_rn(amplitude);
#else
    const float a = (float)amplitude;
#endif
    return d_fdiv(f0_mul(a, (float)amplitude_offset), max_amp);
}

// The curve value of every bin whose cached_bark_cos_omega is `cos_omega`.  The reference evaluates it once per run of
// equal cos_omega values (audio.rs:201-208) and writes it to the whole run; evaluated per bin, equal inputs give the
// same value.
LWB_HD float d_floor0_value(const float *cosc, int order, float common, uint32_t amplitude_offset, float cos_omega)
{
    int pu, qu;
    float p, q;
    if (order & 1) {                                              // audio.rs:175-181
        pu = (order - 3) / 2;
        qu = (order - 1) / 2;
        p = f0_sub(1.0f, f0_mul(cos_omega, cos_omega));
        q = 0.25f;
    } else {                                                      // audio.rs:182-187
        pu = qu = (order - 2) / 2;
        p = f0_mul(f0_sub(1.0f, cos_omega), 0.5f);                // x / 2.0 == x * 0.5: both round x / 2 once
        q = f0_mul(f0_add(1.0f, cos_omega), 0.5f);
    }
    for (int j = 0; j <= pu; j++) {                               // audio.rs:189-192: p *= 4.0 * pm * pm
        const float pm = f0_sub(cosc[2 * j + 1], cos_omega);
        p = f0_mul(p, f0_mul(f0_mul(4.0f, pm), pm));
    }
    for (int j = 0; j <= qu; j++) {                               // audio.rs:193-196
        const float qm = f0_sub(cosc[2 * j], cos_omega);
        q = f0_mul(q, f0_mul(f0_mul(4.0f, qm), qm));
    }
    // audio.rs:198-199
    return d_expf(f0_mul(0.11512925f, f0_sub(d_fdiv(common, d_fsqrt(f0_add(p, q))), (float)amplitude_offset)));
}

// A floor-0 record of one row (LWB_FLOOR_ZERO): the amplitude and the coefficient cosines in the row's floor1_y words.
LWB_HD uint64_t d_floor0_amplitude(const uint32_t *rec) { return (uint64_t)rec[0] | ((uint64_t)rec[1] << 32); }

#if defined(__CUDACC__)
constexpr int kF0Threads = 256;
constexpr int kF0Rows = kF0Threads / 32;        // one warp per row

// grid = ceil(n_rows / kF0Rows), row r = (packet ordinal in pkts) * C + channel.  Rows of kind LWB_FLOOR_ZERO get their
// curve in `curves`, laid out like the coefficient arena (element p.coeff_off + c * n/2 + bin); a row whose floor has
// no floor-0 description gets the zero curve, like LWB_FLOOR_UNUSED (audio.rs:1021-1024).  Other rows are not touched.
__global__ void __launch_bounds__(kF0Threads)
k_floor0_curves(const DevPacket *__restrict__ pkts, uint32_t n_rows, int C, const uint8_t *__restrict__ floor_kind,
                const uint32_t *__restrict__ floor1_y, float *__restrict__ curves)
{
    __shared__ float s_c[kF0Rows][LWB_MAX_POSTS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t row = blockIdx.x * kF0Rows + warp;
    if (row >= n_rows) return;                                    // (whole warps: no block-wide barrier below)
    const uint32_t pk = row / (uint32_t)C, c = row - pk * (uint32_t)C;
    const DevPacket &p = pkts[pk];
    const uint64_t frow = p.pkt_index * (uint64_t)C + c;
    if (floor_kind[frow] != LWB_FLOOR_ZERO) return;
    const int n2 = p.n >> 1;
    float *out = curves + p.coeff_off + (uint64_t)c * n2;
    const DevSetup &su = *p.setup;
    const int fi = su.mappings[p.mapping].floor_of_channel[c];
    const DevFloor0 *f = su.floor0 ? su.floor0 + fi : nullptr;
    if (!f || !f->order) {
        for (int k = lane; k < n2; k += 32) out[k] = 0.f;
        return;
    }
    const uint32_t *rec = floor1_y + frow * LWB_MAX_POSTS;
    const int order = f->order;
    for (int j = lane; j < order; j += 32) s_c[warp][j] = __uint_as_float(rec[2 + j]);
    const float common = d_floor0_common(d_floor0_amplitude(rec), f->amplitude_offset, f->max_amp);
    __syncwarp();
    const float *__restrict__ bark = f->bark_cos_omega[p.blockflag ? 1 : 0];
    for (int k = lane; k < n2; k += 32) out[k] = d_floor0_value(s_c[warp], order, common, f->amplitude_offset, __ldg(bark + k));
}
#endif

}  // namespace lwb
