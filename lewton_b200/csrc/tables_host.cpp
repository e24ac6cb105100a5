// tables_host.cpp -- host-side constants of the synthesis path.
//
// (1) CachedBlocksizeDerived::from_blocksize (lewton src/header_cached.rs:33-110): the IMDCT
//     twiddles A/B/C, the bit-reverse table and the Vorbis window slope.  They are evaluated on
//     the HOST with libm's sinf/cosf -- exactly what Rust's f32::sin/cos call on Linux -- in the
//     reference's f32 expression order, and uploaded; the kernels never call sin/cos, so the
//     device result cannot depend on CUDA's math library.
// (2) floor-1 neighbour indices (src/audio.rs:253-292): they depend only on the x-list, so they
//     are resolved once per setup instead of once per packet.
//
// Compile without contraction (-ffp-contract=off): one rounding per operation as written.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "lwb_common.h"

namespace lwb {

static const float kPi = 3.14159265358979323846f;   // std::f32::consts::PI

// header_cached.rs:43-54
static float window_slope_at(uint32_t x, uint32_t n)
{
    const float inner = std::sin(0.5f * kPi * (static_cast<float>(x) + 0.5f) / static_cast<float>(n));
    return std::sin(0.5f * kPi * inner * inner);
}

// lib.rs:174-176 (u32::reverse_bits)
static uint32_t reverse_bits32(uint32_t v)
{
    v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
    v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
    v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
    return (v >> 16) | (v << 16);
}

int generate_tables(int bs, float *a, float *b, float *c, float *window, uint32_t *bitrev)
{
    if (bs < 6 || bs > 13) return LWB_ERR_INVALID;
    const uint32_t n = 1u << bs;
    const float nf = static_cast<float>(n);
    if (window) {
        // header_cached.rs:56-62 generate_window(n / 2)
        for (uint32_t i = 0; i < n / 2; i++) window[i] = window_slope_at(i, n / 2);
    }
    // header_cached.rs:64-99
    const float step_a = 4.0f * kPi / nf;
    const float step_b = 0.5f * kPi / nf;
    const float step_c = 2.0f * kPi / nf;
    for (uint32_t k = 0; k < n / 4; k++) {
        const float ka = static_cast<float>(k) * step_a;
        const float kb = static_cast<float>(2 * k + 1) * step_b;
        if (a) {
            a[2 * k] = std::cos(ka);
            a[2 * k + 1] = -std::sin(ka);
        }
        if (b) {
            b[2 * k] = std::cos(kb) * 0.5f;
            b[2 * k + 1] = std::sin(kb) * 0.5f;
        }
    }
    if (c) {
        for (uint32_t k = 0; k < n / 8; k++) {
            const float kc = static_cast<float>(2 * k + 1) * step_c;
            c[2 * k] = std::cos(kc);
            c[2 * k + 1] = -std::sin(kc);
        }
    }
    if (bitrev) {
        // header_cached.rs:101-110
        for (uint32_t i = 0; i < n / 8; i++)
            bitrev[i] = (reverse_bits32(i) >> (32 - bs + 3)) << 2;
    }
    return LWB_OK;
}

// Fills sorted order (header.rs:887-889) and the low/high neighbour of every post i >= 2
// (audio.rs:253-292: the closest smaller / larger x among posts 0..i).  Returns LWB_OK, or
// LWB_ERR_BAD_FORMAT for lists the header parser cannot produce (post 0 not at x = 0: it always
// makes [0, 1 << rangebits, ...], header.rs:877-879; duplicates, :890-901) or for which the
// reference's neighbour search would panic.  Post 0 at x = 0 is what lets every kernel start the
// curve at its first flagged post: render_line covers bins from lx = 0 (audio.rs:532-541).
int prepare_floor1(const lwb_floor_desc &d, DevFloor1 *out)
{
    std::memset(out, 0, sizeof(*out));
    out->type = d.floor_type;
    if (d.floor_type != LWB_FLOOR_TYPE_ONE) return LWB_OK;
    const int np = d.floor1_values;
    if (np < 2 || np > LWB_MAX_POSTS) return LWB_ERR_BAD_FORMAT;
    if (d.floor1_multiplier < 1 || d.floor1_multiplier > 4) return LWB_ERR_BAD_FORMAT;
    if (d.floor1_x_list[0] != 0) return LWB_ERR_BAD_FORMAT;
    out->mult = d.floor1_multiplier;
    out->nposts = static_cast<uint8_t>(np);
    for (int i = 0; i < np; i++) {
        if (d.floor1_x_list[i] > 32768u) return LWB_ERR_BAD_FORMAT;   // rangebits is 4 bits
        out->x[i] = static_cast<uint16_t>(d.floor1_x_list[i]);
    }
    int order[LWB_MAX_POSTS];
    for (int i = 0; i < np; i++) order[i] = i;
    for (int i = 1; i < np; i++) {          // stable insertion sort by x
        const int cur = order[i];
        int j = i;
        while (j > 0 && d.floor1_x_list[order[j - 1]] > d.floor1_x_list[cur]) {
            order[j] = order[j - 1];
            j--;
        }
        order[j] = cur;
    }
    for (int i = 0; i < np; i++) {
        if (i && d.floor1_x_list[order[i]] == d.floor1_x_list[order[i - 1]]) return LWB_ERR_BAD_FORMAT;
        out->sorted[i] = static_cast<uint8_t>(order[i]);
    }
    for (int i = 2; i < np; i++) {
        const uint32_t xi = d.floor1_x_list[i];
        int lo = -1, hi = -1;
        for (int j = 0; j < i; j++) {
            const uint32_t xj = d.floor1_x_list[j];
            if (xj < xi && (lo < 0 || xj > d.floor1_x_list[lo])) lo = j;
            if (xj > xi && (hi < 0 || xj < d.floor1_x_list[hi])) hi = j;
        }
        if (lo < 0 || hi < 0) return LWB_ERR_BAD_FORMAT;
        out->lo[i] = static_cast<uint8_t>(lo);
        out->hi[i] = static_cast<uint8_t>(hi);
    }
    return LWB_OK;
}

}  // namespace lwb
