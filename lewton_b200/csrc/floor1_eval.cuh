// floor1_eval.cuh -- floor type 1 evaluation (audio.rs:354-555), integer only.  Host+device (LWB_HD) so
// that tests/emu/floor1_emu.cpp can run exactly this source on the CPU against the oracle.
#pragma once
#include "kernel_long.cuh"      // LWB_HD
#include "lwb_common.h"

namespace lwb {

// ---------------------------------------------------------------------------------------------
// floor-1, audio.rs:354-435 -- run by one thread per (packet, channel); <= 65 posts, serial
// ---------------------------------------------------------------------------------------------
LWB_HD uint32_t d_render_point(uint32_t x0, uint32_t y0, uint32_t x1,
                                                   uint32_t y1, uint32_t x)
{
    // audio.rs:354-367, u32/i32 wrapping like a release build
    const int32_t dy = (int32_t)(y1 - y0);
    const uint32_t adx = x1 - x0;
    const uint32_t ady = (uint32_t)(dy < 0 ? -dy : dy);
    const uint32_t off = (ady * (x - x0)) / adx;
    return dy < 0 ? y0 - off : y0 + off;
}

// Writes the flagged posts in x order as (sx, sy = y * multiplier); returns their count
// (+1 if a flat tail to n2 was appended, audio.rs:546-547).
LWB_HD int d_floor1_posts(const DevFloor1 &fl, const uint32_t *__restrict__ y_in, int n2,
                              uint16_t *sx, uint16_t *sy)
{
    uint32_t fy[LWB_MAX_POSTS];
    uint64_t flag_lo = 3;        // posts 0..63
    bool flag64 = false;         // post 64
    const int np = fl.nposts;
    const int32_t range = fl.mult == 1 ? 256 : fl.mult == 2 ? 128 : fl.mult == 3 ? 86 : 64;
    fy[0] = y_in[0];
    fy[1] = y_in[1];
    for (int i = 2; i < np; i++) {           // audio.rs:401-429
        const int li = fl.lo[i], hi = fl.hi[i];
        const int32_t predicted =
            (int32_t)d_render_point(fl.x[li], fy[li], fl.x[hi], fy[hi], fl.x[i]);
        const int32_t val = (int32_t)y_in[i];
        const int32_t highroom = range - predicted;
        const int32_t lowroom = predicted;
        const int32_t room = (highroom < lowroom ? highroom : lowroom) * 2;
        if (val > 0) {
            flag_lo |= (1ull << li) | (1ull << hi);     // li, hi < i <= 64
            if (i < 64) flag_lo |= 1ull << i; else flag64 = true;
            int32_t r;
            if (val >= room) {
                r = highroom > lowroom ? predicted + val - lowroom : predicted - val + highroom - 1;
            } else {
                const int32_t t = (val % 2 == 1) ? (-val - 1) : val;
                r = predicted + (t >> 1);
            }
            fy[i] = (uint32_t)r;
        } else {
            fy[i] = (uint32_t)predicted;
        }
    }
    int m = 0;
    uint32_t hx = 0, hy = 0;
    for (int j = 0; j < np; j++) {           // audio.rs:528-545, in sorted order
        const int si = fl.sorted[j];
        const bool flagged = si < 64 ? ((flag_lo >> si) & 1ull) : flag64;
        if (j == 0 || flagged) {
            uint32_t v = fy[si];
            if (v > (uint32_t)range - 1) v = (uint32_t)range - 1;     // audio.rs:431-433
            hy = v * fl.mult;
            hx = fl.x[si];
            sx[m] = (uint16_t)hx;
            sy[m] = (uint16_t)hy;
            m++;
        }
    }
    if (hx < (uint32_t)n2) {                 // audio.rs:546-547 flat tail
        sx[m] = (uint16_t)n2;
        sy[m] = (uint16_t)hy;
        m++;
    }
    return m;
}

// Value of the rendered integer curve at bin k: the closed form of render_line (audio.rs:503-524):
// y0 + sign(dy) * floor(|dy| * (k - x0) / adx) for the segment [x0, x1) containing k.
LWB_HD uint32_t d_floor1_y_at(const uint16_t *sx, const uint16_t *sy, int m, int k)
{
    int lo = 0, hi = m - 1;                  // sx[lo] <= k < sx[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if ((int)sx[mid] <= k) lo = mid; else hi = mid;
    }
    const int x0 = sx[lo], x1 = sx[lo + 1];
    const int y0 = sy[lo], y1 = sy[lo + 1];
    const int dy = y1 - y0;
    const int ady = dy < 0 ? -dy : dy;
    const int off = (ady * (k - x0)) / (x1 - x0);
    return (uint32_t)(dy < 0 ? y0 - off : y0 + off);
}

// One flagged segment [sx[seg], sx[seg + 1]) of the curve, rendered the way the reference does
// (render_line, audio.rs:503-524: integer DDA, one division per segment), clipped to n2 bins
// (audio.rs:548-550).  Curve values fit a byte: posts are clamped to range - 1 and range * multiplier <= 256.
LWB_HD void d_floor1_render_segment(const uint16_t *sx, const uint16_t *sy, int seg, int n2, uint8_t *curve)
{
    const int x0 = sx[seg], x1 = sx[seg + 1];
    if (x0 >= n2) return;
    const int y0 = sy[seg], y1 = sy[seg + 1];
    const int dy = y1 - y0, adx = x1 - x0;
    int ady = dy < 0 ? -dy : dy;
    const int base = dy / adx;
    const int sgn = dy < 0 ? base - 1 : base + 1;
    ady -= (base < 0 ? -base : base) * adx;
    const int end = x1 < n2 ? x1 : n2;
    int y = y0, err = 0;
    curve[x0] = (uint8_t)y;
    for (int x = x0 + 1; x < end; x++) {
        err += ady;
        if (err >= adx) { err -= adx; y += sgn; }
        else y += base;
        curve[x] = (uint8_t)y;
    }
}

// ---- division-free closed form (d_floor1_pack_segment, k_floor1_segments) ----------------------
// floor(N / adx) for N = |dy| * (k - x0) < 2^20 (|dy| < 2^8, k - x0 < n/2 <= 2^12) by one multiply-high, no
// division anywhere:  M = floor((2^(32+s) - 1) / adx) + 1,  floor(N / adx) == mulhi(N, M) >> s  whenever
// N * adx < 2^(32+s)  (M * adx = 2^(32+s) + e with 0 < e <= adx, and the error term N * e / (adx * 2^(32+s)) stays
// below 1 / adx).  s = 0 covers every adx <= 4096; longer segments (x lists may reach 2^15) take s = 12, where M
// still fits 32 bits.  adx == 1: the only bin of the segment has N == 0.
LWB_HD uint32_t d_floor1_magic(int adx, int *shift)
{
    *shift = adx > 4096 ? 12 : 0;
    if (adx < 2) return 1u;
    const uint64_t one = 1ull << (32 + *shift);
    return (uint32_t)((one - 1) / (uint64_t)adx + 1);
}

LWB_HD uint32_t d_mulhi_u32(uint32_t a, uint32_t b)
{
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// One flagged segment [x0, x1) of a floor curve, packed for per-bin evaluation (k_prologue_fused), laid out so
// that a bin costs as few instructions as possible:
//   .x = multiply-high magic of adx
//   .y = x1 << 16 | y0 << 8 | (shift ? 2 : 0) | (dy < 0 ? 1 : 0)     -- "bin k is past this segment" is the single
//                                                                       unsigned compare (k << 16 | 0xffff) >= .y
//   .z = |dy|            .w = -(|dy| * x0)                           -- |dy| * (k - x0) is one multiply-add
// y(k) = y0 +- (mulhi(|dy| * (k - x0), magic) >> shift): the closed form of render_line (audio.rs:503-524).
struct Seg4 { uint32_t x, y, z, w; };
// magic_tab: d_floor1_magic of every adx in [0, 32768] (kFloor1MagicEntries words), built once per context -- the
// 64-bit division behind it is ~150 instructions on the device, and a row has up to 66 segments; nullptr: compute it.
constexpr int kFloor1MagicEntries = 32769;
LWB_HD Seg4 d_floor1_pack_segment(const uint16_t *sx, const uint16_t *sy, int j, const uint32_t *magic_tab = nullptr)
{
    const int adx = (int)sx[j + 1] - (int)sx[j];
    int sh = adx > 4096 ? 12 : 0;
    const uint32_t mg = magic_tab && adx >= 0 ? magic_tab[adx] : d_floor1_magic(adx, &sh);
    const int y0 = sy[j] & 255, dy = (int)(sy[j + 1] & 255) - y0;
    const uint32_t ady = (uint32_t)(dy < 0 ? -dy : dy);
    Seg4 s;
    s.x = mg;
    s.y = ((uint32_t)sx[j + 1] << 16) | ((uint32_t)y0 << 8) | (sh ? 2u : 0u) | (dy < 0 ? 1u : 0u);
    s.z = ady;
    s.w = 0u - ady * (uint32_t)sx[j];
    return s;
}
LWB_HD bool d_floor1_seg_past(const Seg4 &s, int k) { return (((uint32_t)k << 16) | 0xffffu) >= s.y; }
template <bool SHIFT>
LWB_HD uint32_t d_floor1_seg_y(const Seg4 &s, int k)
{
    uint32_t q = d_mulhi_u32(s.z * (uint32_t)k + s.w, s.x);
    if (SHIFT) q >>= (s.y & 2u) ? 12 : 0;
    const uint32_t y0 = (s.y >> 8) & 255u, neg = 0u - (s.y & 1u);
    return y0 + ((q ^ neg) - neg);
}

}  // namespace lwb
