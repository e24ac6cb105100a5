// floor0_emu.cpp -- TEST INFRASTRUCTURE: the floor-0 source the GPU compiles (lewton_b200/csrc/kernel_floor0.cuh), run on
// the host: the restated expf, the FMA-free division and square root, and the per-bin curve of one row.
#include <cmath>
#include <cstring>

#include "../../lewton_b200/csrc/kernel_floor0.cuh"

static uint32_t bits(float f)
{
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return u;
}
static float flt(uint32_t u)
{
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}
// equal bit patterns, or both NaN (the payload is not part of the result)
static bool same(float a, float b) { return bits(a) == bits(b) || (std::isnan(a) && std::isnan(b)); }

// Inputs in [lo, hi) (as bit patterns) where d_expf (op 0) / d_fsqrt (op 1) differs from the host's expf / sqrtf;
// *first = the first of them.
extern "C" uint64_t lwb_emu_unary_mismatches(int op, uint64_t lo, uint64_t hi, uint32_t *first)
{
    uint64_t bad = 0;
    for (uint64_t u = lo; u < hi; u++) {
        const float x = flt((uint32_t)u);
        const bool ok = op == 0 ? same(lwb::d_expf(x), expf(x)) : same(lwb::d_fsqrt(x), sqrtf(x));
        if (!ok && bad++ == 0) *first = (uint32_t)u;
    }
    return bad;
}

// n pseudo-random pairs (xorshift from seed; every third a from a narrow exponent window around b's, so that quotients
// near 1, subnormal and overflowing ones all occur) where d_fdiv differs from a / b; first pair in out[0..1].
extern "C" uint64_t lwb_emu_div_mismatches(uint64_t seed, uint64_t n, uint32_t *first)
{
    uint64_t s = seed | 1, bad = 0;
    auto next = [&]() {
        s ^= s << 13;
        s ^= s >> 7;
        s ^= s << 17;
        return s;
    };
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t r = next();
        uint32_t ua = (uint32_t)r, ub = (uint32_t)(r >> 32);
        if (i % 3 == 0) ua = (ua & 0x807fffffu) | (((ub >> 23) & 0xffu) + (uint32_t)(r % 9) - 4) % 255u << 23;
        const float a = flt(ua), b = flt(ub);
        if (!same(lwb::d_fdiv(a, b), a / b) && bad++ == 0) {
            first[0] = ua;
            first[1] = ub;
        }
    }
    return bad;
}

// One row of k_floor0_curves: n2 bins of the curve of a floor (order, amplitude_bits, amplitude_offset) with record
// (amplitude, cosc) over the bark table `bark` (n2 values).
extern "C" void lwb_emu_floor0_row(int order, int amplitude_bits, int amplitude_offset, uint64_t amplitude, const float *cosc,
                                   const float *bark, int n2, float *out)
{
    const float common = lwb::d_floor0_common(amplitude, (uint32_t)amplitude_offset, lwb::d_floor0_max_amp(amplitude_bits));
    for (int k = 0; k < n2; k++) out[k] = lwb::d_floor0_value(cosc, order, common, (uint32_t)amplitude_offset, bark[k]);
}
