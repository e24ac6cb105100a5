// floor1_emu.cpp -- TEST INFRASTRUCTURE: the floor-1 evaluation source the GPU compiles
// (lewton_b200/csrc/floor1_eval.cuh + prepare_floor1 of tables_host.cpp), run on the host:
// post unwrap, closed-form curve and the DDA segment render, for the oracle to check.
#include <cstring>
#include <vector>

#include "../../lewton_b200/csrc/floor1_eval.cuh"
#include "../../lewton_b200/csrc/tables_host.cpp"

extern "C" int lwb_emu_floor1(int mult, const uint32_t *xs, int nposts, const uint32_t *y, int n2,
                              uint32_t *curve_closed, uint8_t *curve_render, uint8_t *curve_packed)
{
    lwb_floor_desc d;
    std::memset(&d, 0, sizeof(d));
    d.floor_type = LWB_FLOOR_TYPE_ONE;
    d.floor1_multiplier = (uint8_t)mult;
    d.floor1_values = (uint8_t)nposts;
    for (int i = 0; i < nposts; i++) d.floor1_x_list[i] = xs[i];
    lwb::DevFloor1 fl;
    const int rc = lwb::prepare_floor1(d, &fl);
    if (rc) return rc;
    uint16_t sx[LWB_MAX_POSTS + 1], sy[LWB_MAX_POSTS + 1];
    const int m = lwb::d_floor1_posts(fl, y, n2, sx, sy);
    for (int k = 0; k < n2; k++) curve_closed[k] = lwb::d_floor1_y_at(sx, sy, m, k);
    std::memset(curve_render, 0xee, (size_t)n2);
    for (int seg = 0; seg + 1 < m; seg++) lwb::d_floor1_render_segment(sx, sy, seg, n2, curve_render);
    // the packed-segment evaluation of k_prologue_fused: per bin, segment advanced without branches
    {
        lwb::Seg4 tab[LWB_MAX_POSTS + 2];
        uint16_t sx2[LWB_MAX_POSTS + 1], sy2[LWB_MAX_POSTS + 1];
        const int m2 = lwb::d_floor1_posts(fl, y, n2, sx2, sy2);
        for (int j = 0; j + 1 < m2; j++) tab[j] = lwb::d_floor1_pack_segment(sx2, sy2, j);
        tab[m2 - 1] = tab[m2 - 2];                     // sentinel read past the last segment (never selected: x1 >= n2)
        int seg = 0;
        for (int k = 0; k < n2; k++) {
            seg += lwb::d_floor1_seg_past(tab[seg], k);
            curve_packed[k] = (uint8_t)lwb::d_floor1_seg_y<true>(tab[seg], k);
        }
    }
    return 0;
}

// exactness of the multiply-high division d_floor1_pack_segment packs into each segment: every adx up to 2^15, every |dy|, dense t
extern "C" long lwb_emu_magic_mismatches(int adx_lo, int adx_hi)
{
    long bad = 0;
    for (int adx = adx_lo; adx <= adx_hi; adx++) {
        int sh;
        const uint32_t mg = lwb::d_floor1_magic(adx, &sh);
        if (adx > 4200 && adx % 61 && adx != adx_hi) continue;   // long segments: a sample of the lengths, all of the short ones
        for (uint32_t ady = 0; ady < 256; ady++)
            for (uint32_t t = 0; t < 4096; t += (t < 64 || t > 4000) ? 1 : 7) {
                if (adx == 1 && t) break;                      // a one-bin segment only ever sees t == 0
                const uint32_t nn = ady * t;
                if ((lwb::d_mulhi_u32(nn, mg) >> sh) != nn / (uint32_t)adx) bad++;
            }
    }
    return bad;
}
