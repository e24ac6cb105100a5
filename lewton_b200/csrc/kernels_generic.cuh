// kernels_generic.cuh -- the general synthesis path: any blocksize 6..13, any channel count,
// mixed short/long sequences, all output formats.  Four kernels, fully parallel over packets:
//
//   k_prologue  : inverse coupling -> floor-1 render -> floor x residue   (audio.rs:991-1039)
//   k_imdct     : inverse MDCT of one (packet, channel) block in shared memory (imdct.rs:291-659)
//   k_overlap   : window / overlap-add / slice / sample conversion         (audio.rs:1079-1157)
//   k_save_state: PreviousWindowRight update                                (audio.rs:1121,1154)
//
// Bandwidth: this path round-trips the spectrum and the un-windowed IMDCT output through HBM
// (about 32 B per output sample instead of the algorithmic 8); the fused kernel in
// kernel_long.cuh is the hot path for the headline configuration, this one is the general
// fallback every configuration is correct on.
//
// Arithmetic rules (parity with the reference): binary32, round-to-nearest, no FMA contraction
// (-fmad=false), denormals kept (-ftz=false); every butterfly uses the reference's operand order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernel_long.cuh"
#include "lwb_common.h"
#include "floor1_eval.cuh"

namespace lwb {

__constant__ float c_inverse_db[256] = {
#include "floor1_inverse_db.inc"
};

// audio.rs:762-777, branch-free.  With s = (a > 0), t = (m > 0) (both false for NaN, like the reference's `> 0.`):
//   v = m + (t == s ? -a : a)   -- m - a and m + (-a) are the same IEEE operation --
//   s: (m, a) <- (m, v);  !s: (m, a) <- (v, m)
__device__ __forceinline__ void d_inverse_couple(float &m, float &a)
{
    const float m0 = m, a0 = a;
    const bool s = a0 > 0.f, t = m0 > 0.f;
    const float v = __fadd_rn(m0, (t == s) ? -a0 : a0);
    m = s ? m0 : v;
    a = s ? v : m0;
}
// the same on each of four consecutive bins
__device__ __forceinline__ void d_inverse_couple(float4 &m, float4 &a)
{
    d_inverse_couple(m.x, a.x); d_inverse_couple(m.y, a.y);
    d_inverse_couple(m.z, a.z); d_inverse_couple(m.w, a.w);
}
// floor x residue of four consecutive bins (audio.rs:1035-1037)
__device__ __forceinline__ float4 d_floor_mul(float4 f, float4 r)
{
    return make_float4(__fmul_rn(f.x, r.x), __fmul_rn(f.y, r.y), __fmul_rn(f.z, r.z), __fmul_rn(f.w, r.w));
}
// At most one coupling step over two channels (r0, r1: channels 0 and 1); swapped: (magnitude, angle) = (1, 0).
// T is float or float4.
template <typename T>
__device__ __forceinline__ void d_inverse_couple_stereo(int nsteps, bool swapped, T &r0, T &r1)
{
    if (nsteps == 1) {
        if (swapped) d_inverse_couple(r1, r0);
        else d_inverse_couple(r0, r1);
    }
}
// The nsteps coupling steps of mp, in reverse (audio.rs:991-1002), on one bin of up to 8 channels held in registers.
// The channel indices are dynamic, so each step reads and writes its pair through predicated selects.
__device__ __forceinline__ void d_inverse_couple_regs(float (&r)[8], const DevMapping &mp, int nsteps)
{
    for (int s = nsteps - 1; s >= 0; s--) {
        const int mi = mp.mag[s], ai = mp.ang[s];
        float mv = 0.f, av = 0.f;
#pragma unroll
        for (int c = 0; c < 8; c++) { if (c == mi) mv = r[c]; if (c == ai) av = r[c]; }
        d_inverse_couple(mv, av);
#pragma unroll
        for (int c = 0; c < 8; c++) { if (c == mi) r[c] = mv; if (c == ai) r[c] = av; }
    }
}

constexpr int kPrologueThreads = 256;
constexpr int kPrologueGroup = 8;            // channels whose floor posts sit in smem at once
// dynamic shared memory of k_prologue: one curve byte per bin for up to 8 channels of the largest block
inline size_t prologue_smem(int channels, int blocksize_1) { return (size_t)(channels < kPrologueGroup ? channels : kPrologueGroup) << (blocksize_1 - 1); }

// The floor value of a row of kind `kind` (not LWB_FLOOR_ONE) at coefficient element e: the host's dense curve, the
// curve k_floor0_curves rendered (zero_floor; nullptr: the row acts as unused), or 0 (audio.rs:1021-1024).
__device__ __forceinline__ float d_floor_other(int kind, const float *__restrict__ dense_floor, const float *__restrict__ zero_floor, uint64_t e)
{
    if (kind == LWB_FLOOR_DENSE) return dense_floor[e];
    if (kind == LWB_FLOOR_ZERO && zero_floor) return zero_floor[e];
    return 0.f;
}

// grid.x = packets.  spec[packet] = [channels][n/2] receives floor x decoupled residue.
__global__ void __launch_bounds__(kPrologueThreads)
k_prologue(const DevPacket *__restrict__ pkts, const float *__restrict__ residue,
           const float *__restrict__ dense_floor, const uint8_t *__restrict__ floor_kind,
           const uint32_t *__restrict__ floor1_y, float *__restrict__ spec, const float *__restrict__ zero_floor)
{
    const DevPacket &p = pkts[blockIdx.x];
    const DevSetup &su = *p.setup;
    const DevMapping &mp = su.mappings[p.mapping];
    const int C = p.channels;
    const int n2 = p.n >> 1;
    const float *res = residue + p.coeff_off;
    float *out = spec + p.coeff_off;
    const int nsteps = mp.n_coupling;

    __shared__ uint16_t s_x[kPrologueGroup][LWB_MAX_POSTS + 1];
    __shared__ uint16_t s_y[kPrologueGroup][LWB_MAX_POSTS + 1];
    __shared__ int s_m[kPrologueGroup];
    const uint8_t *kinds = floor_kind + p.pkt_index * C;

    if (C <= kPrologueGroup) {
        // Up to 8 channels: the floor curves are rendered once into shared memory (one byte per bin) and a
        // single pass over the bins does the rest, so every value crosses the memory system once.
        //   a. posts: one lane per channel, serial over <= 65 posts (audio.rs:391-435);
        //   b. curve: warp w renders channel w, one flagged segment per lane, with the reference's own
        //      integer DDA (render_line, audio.rs:503-524) -- no search and no division per bin;
        //   c. bins: load the residues, inverse-couple them in registers (steps in reverse,
        //      audio.rs:991-1002), multiply by the floor (audio.rs:1006-1039), store.
        extern __shared__ uint8_t s_curve_raw[];            // [C][n2] bytes: the host passes min(C, 8) * blocksize_1 / 2
        uint8_t *s_curve = s_curve_raw;
        const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (lane == 0 && w < C && kinds[w] == LWB_FLOOR_ONE) {
            const DevFloor1 &fl = su.floors[mp.floor_of_channel[w]];
            s_m[w] = d_floor1_posts(fl, floor1_y + (p.pkt_index * C + w) * LWB_MAX_POSTS, n2, s_x[w], s_y[w]);
        }
        __syncwarp();
        if (w < C && kinds[w] == LWB_FLOOR_ONE)
            for (int seg = lane; seg + 1 < s_m[w]; seg += 32) d_floor1_render_segment(s_x[w], s_y[w], seg, n2, s_curve + (size_t)w * n2);
        __syncthreads();
        if (C == 2 && nsteps <= 1) {
            // the common stereo shape: at most one coupling step, no register-array juggling
            const bool swapped = nsteps == 1 && mp.mag[0] == 1;       // (magnitude, angle) = (1, 0)
            const int k0 = kinds[0], k1 = kinds[1];
            for (int k = threadIdx.x; k < n2; k += kPrologueThreads) {
                float r0 = res[k], r1 = res[(size_t)n2 + k];
                d_inverse_couple_stereo(nsteps, swapped, r0, r1);
                const float f0 = k0 == LWB_FLOOR_ONE ? c_inverse_db[s_curve[k]] : d_floor_other(k0, dense_floor, zero_floor, p.coeff_off + k);
                const float f1 = k1 == LWB_FLOOR_ONE ? c_inverse_db[s_curve[(size_t)n2 + k]]
                                                     : d_floor_other(k1, dense_floor, zero_floor, p.coeff_off + (size_t)n2 + k);
                out[k] = __fmul_rn(f0, r0);                            // audio.rs:1035-1037
                out[(size_t)n2 + k] = __fmul_rn(f1, r1);
            }
            return;
        }
        for (int k = threadIdx.x; k < n2; k += kPrologueThreads) {
            float r[8];
#pragma unroll
            for (int c = 0; c < 8; c++) r[c] = c < C ? res[(size_t)c * n2 + k] : 0.f;
            d_inverse_couple_regs(r, mp, nsteps);
#pragma unroll
            for (int c = 0; c < 8; c++) {
                if (c < C) {
                    const int kind = kinds[c];
                    const float f = kind == LWB_FLOOR_ONE ? c_inverse_db[s_curve[(size_t)c * n2 + k]]
                                                          : d_floor_other(kind, dense_floor, zero_floor, p.coeff_off + (size_t)c * n2 + k);
                    out[(size_t)c * n2 + k] = __fmul_rn(f, r[c]);
                }
            }
        }
        return;
    }

    // more than 8 channels: two passes through `out`
    // 1. inverse coupling, steps in reverse (audio.rs:991-1002).  Every thread owns its bins
    //    through all steps, so the working copy in `out` needs no synchronisation.
    for (int k = threadIdx.x; k < n2; k += kPrologueThreads) {
        for (int c = 0; c < C; c++) out[(size_t)c * n2 + k] = res[(size_t)c * n2 + k];
        for (int s = nsteps - 1; s >= 0; s--) {
            float mv = out[(size_t)mp.mag[s] * n2 + k], av = out[(size_t)mp.ang[s] * n2 + k];
            d_inverse_couple(mv, av);
            out[(size_t)mp.mag[s] * n2 + k] = mv;
            out[(size_t)mp.ang[s] * n2 + k] = av;
        }
    }

    // 2. floor curve x residue (audio.rs:1006-1039), kPrologueGroup channels at a time
    for (int c0 = 0; c0 < C; c0 += kPrologueGroup) {
        __syncthreads();
        const int w = threadIdx.x >> 5;
        if ((threadIdx.x & 31) == 0 && c0 + w < C && kinds[c0 + w] == LWB_FLOOR_ONE) {
            const int c = c0 + w;
            const DevFloor1 &fl = su.floors[mp.floor_of_channel[c]];
            s_m[w] = d_floor1_posts(fl, floor1_y + (p.pkt_index * C + c) * LWB_MAX_POSTS, n2,
                                    s_x[w], s_y[w]);
        }
        __syncthreads();
        for (int g = 0; g < kPrologueGroup && c0 + g < C; g++) {
            const int c = c0 + g;
            const int kind = kinds[c];
            float *oc = out + (size_t)c * n2;
            for (int k = threadIdx.x; k < n2; k += kPrologueThreads) {
                const float f = kind == LWB_FLOOR_ONE ? c_inverse_db[d_floor1_y_at(s_x[g], s_y[g], s_m[g], k) & 255u]
                                                      : d_floor_other(kind, dense_floor, zero_floor, p.coeff_off + (size_t)c * n2 + k);
                oc[k] = __fmul_rn(f, oc[k]);           // audio.rs:1035-1037
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// inverse MDCT, imdct.rs:291-659, stage by stage in shared memory
// ---------------------------------------------------------------------------------------------
// imdct.rs:201-232, z7 = &zm7[7]
__device__ __forceinline__ void d_iter_54(float *z7)
{
    const float k00 = __fsub_rn(z7[0], z7[-4]);
    const float y0 = __fadd_rn(z7[0], z7[-4]);
    const float y2 = __fadd_rn(z7[-2], z7[-6]);
    const float k22 = __fsub_rn(z7[-2], z7[-6]);
    z7[0] = __fadd_rn(y0, y2);
    z7[-2] = __fsub_rn(y0, y2);
    const float k33 = __fsub_rn(z7[-3], z7[-7]);
    z7[-4] = __fadd_rn(k00, k33);
    z7[-6] = __fsub_rn(k00, k33);
    const float k11 = __fsub_rn(z7[-1], z7[-5]);
    const float y1 = __fadd_rn(z7[-1], z7[-5]);
    const float y3 = __fadd_rn(z7[-3], z7[-7]);
    z7[-1] = __fadd_rn(y1, y3);
    z7[-3] = __fsub_rn(y1, y3);
    z7[-5] = __fsub_rn(k11, k22);
    z7[-7] = __fadd_rn(k11, k22);
}

constexpr int kImdctThreads = 128;

// Steps 0-7 of inverse_mdct (imdct.rs:337-580) for NP independent blocks of one size, cooperatively by NT threads (`tid`
// in [0, NT)) that `sync()` synchronises (a warp, a named-barrier group, or the CTA).  Block q: spectrum X + q * xs (n/2
// coefficients, global or shared; may alias U when NP = 1), buffers U + q * bs and V + q * bs; on return V holds the
// post-step-7 buffer that step 8 (d_imdct_step8) reads.  Literal schedule, including the reference's behaviour for
// n = 64/128.  Every stage first loads the operands of all NP blocks, then computes, then stores, so that a thread has
// NP independent dependency chains in flight instead of one -- the transform is latency-bound for small n, where a
// stage is a single butterfly per lane and each instruction waits on the one before it.
template <int NP, class Sync>
__device__ __forceinline__ void d_imdct_to_v(const DevTables &tb, int n, const float *X, size_t xs, float *U, float *V, int bs,
                                             int tid, int NT, Sync sync)
{
    const int n2 = n >> 1, n4 = n >> 2, n8 = n >> 3;
    const int ld = tb.bs;
    const float *__restrict__ A = tb.a;
    const float *__restrict__ Cc = tb.c;
    // step 0 (imdct.rs:337-371): V <- rotated, reflected spectrum
    for (int t = tid; t < n8; t += NT) {
        const float a0 = A[2 * t], a1 = A[2 * t + 1];
        const int d = n4 - 2 - 2 * t, ao = n4 + 2 * t, e = n2 - 3 - 4 * t;
        const float b0 = A[ao], b1 = A[ao + 1];
        float x0[NP], x2[NP], ne2[NP], ne0[NP];
#pragma unroll
        for (int q = 0; q < NP; q++) {
            const float *Xq = X + q * xs;
            x0[q] = Xq[4 * t]; x2[q] = Xq[4 * t + 2]; ne2[q] = -Xq[e + 2]; ne0[q] = -Xq[e];
        }
#pragma unroll
        for (int q = 0; q < NP; q++) {
            float *Vq = V + q * bs;
            Vq[n2 - 1 - 2 * t] = __fsub_rn(__fmul_rn(x0[q], a0), __fmul_rn(x2[q], a1));
            Vq[n2 - 2 - 2 * t] = __fadd_rn(__fmul_rn(x0[q], a1), __fmul_rn(x2[q], a0));
            Vq[d + 1] = __fsub_rn(__fmul_rn(ne2[q], b0), __fmul_rn(ne0[q], b1));
            Vq[d] = __fadd_rn(__fmul_rn(ne2[q], b1), __fmul_rn(ne0[q], b0));
        }
    }
    sync();
    // step 2 (imdct.rs:385-430): U <- V
    for (int t = tid; t < (n >> 4); t += NT) {
        const int ao = n2 - 8 - 8 * t, hi = n4 + 4 * t, lo = 4 * t;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int o = 2 * h;                  // pair (0,1) uses A[ao+4..5], pair (2,3) A[ao..ao+1]
            const float w0 = A[ao + 4 - 4 * h], w1 = A[ao + 5 - 4 * h];
            float h1[NP], l1[NP], h0[NP], l0[NP];
#pragma unroll
            for (int q = 0; q < NP; q++) {
                const float *Vq = V + q * bs;
                h1[q] = Vq[hi + o + 1]; l1[q] = Vq[lo + o + 1]; h0[q] = Vq[hi + o]; l0[q] = Vq[lo + o];
            }
#pragma unroll
            for (int q = 0; q < NP; q++) {
                float *Uq = U + q * bs;
                const float v1 = __fsub_rn(h1[q], l1[q]), v0 = __fsub_rn(h0[q], l0[q]);
                Uq[hi + o + 1] = __fadd_rn(h1[q], l1[q]);
                Uq[hi + o] = __fadd_rn(h0[q], l0[q]);
                Uq[lo + o + 1] = __fsub_rn(__fmul_rn(v1, w0), __fmul_rn(v0, w1));
                Uq[lo + o] = __fadd_rn(__fmul_rn(v0, w0), __fmul_rn(v1, w1));
            }
        }
    }
    sync();
    // step 3 (imdct.rs:445-477), literal schedule: stage 0, stage 1 (a no-op for n = 64),
    // stages 2..ld-7.  For n = 64/128 this overlaps what ld654 does again below -- the
    // reference's behaviour, kept bit for bit.  Each butterfly is imdct.rs:36-41 / 94-99 / 161-166.
    for (int l = 0; l < 2 || l <= ld - 7; l++) {
        if (l == 1 && n < 128) continue;          // r_loop(lim = n >> 5 = 2): lim >> 2 == 0 iterations
        const int k0 = n >> (l + 2), k1 = 1 << (l + 3);
        const int rbits = ld - l - 4;             // r < n >> (l+4)
        for (int qq = tid; qq < n8; qq += NT) {
            const int r = qq & ((1 << rbits) - 1), s = qq >> rbits;
            const int i = n2 - 1 - k0 * s - 2 * r, lo = i - (k0 >> 1);
            const float w0 = A[r * k1], w1 = A[r * k1 + 1];
            float eh[NP], el[NP], eh1[NP], el1[NP];
#pragma unroll
            for (int q = 0; q < NP; q++) {
                const float *Uq = U + q * bs;
                eh[q] = Uq[i]; el[q] = Uq[lo]; eh1[q] = Uq[i - 1]; el1[q] = Uq[lo - 1];
            }
#pragma unroll
            for (int q = 0; q < NP; q++) {
                float *Uq = U + q * bs;
                const float k00 = __fsub_rn(eh[q], el[q]), k01 = __fsub_rn(eh1[q], el1[q]);
                Uq[i] = __fadd_rn(eh[q], el[q]);
                Uq[i - 1] = __fadd_rn(eh1[q], el1[q]);
                Uq[lo] = __fsub_rn(__fmul_rn(k00, w0), __fmul_rn(k01, w1));
                Uq[lo - 1] = __fadd_rn(__fmul_rn(k01, w0), __fmul_rn(k00, w1));
            }
        }
        sync();
    }
    // imdct.rs:234-288 (ld654): last three stages per 16-float group; NP blocks x (n >> 5) groups share the threads
    {
        const float a2 = A[n >> 3];
        const int groups = n >> 5;
        for (int gq = tid; gq < groups * NP; gq += NT) {
            const int q = NP == 1 ? 0 : gq / groups, g = gq - q * groups;
            float *z = U + q * bs + (n2 - 1 - 16 * g);
            float k00, k11;
            k00 = __fsub_rn(z[0], z[-8]);   k11 = __fsub_rn(z[-1], z[-9]);
            z[0] = __fadd_rn(z[0], z[-8]);  z[-1] = __fadd_rn(z[-1], z[-9]);
            z[-8] = k00;                    z[-9] = k11;
            k00 = __fsub_rn(z[-2], z[-10]); k11 = __fsub_rn(z[-3], z[-11]);
            z[-2] = __fadd_rn(z[-2], z[-10]); z[-3] = __fadd_rn(z[-3], z[-11]);
            z[-10] = __fmul_rn(__fadd_rn(k00, k11), a2);
            z[-11] = __fmul_rn(__fsub_rn(k11, k00), a2);
            k00 = __fsub_rn(z[-12], z[-4]); k11 = __fsub_rn(z[-5], z[-13]);
            z[-4] = __fadd_rn(z[-4], z[-12]); z[-5] = __fadd_rn(z[-5], z[-13]);
            z[-12] = k11;                   z[-13] = k00;
            k00 = __fsub_rn(z[-14], z[-6]); k11 = __fsub_rn(z[-7], z[-15]);
            z[-6] = __fadd_rn(z[-6], z[-14]); z[-7] = __fadd_rn(z[-7], z[-15]);
            z[-14] = __fmul_rn(__fadd_rn(k00, k11), a2);
            z[-15] = __fmul_rn(__fsub_rn(k00, k11), a2);
            d_iter_54(z);
            d_iter_54(z - 8);
        }
    }
    sync();
    // steps 4-6 (imdct.rs:490-528): bit-reverse shuffle U -> V
    for (int qq = tid; qq < (n >> 4); qq += NT) {
        const int d0 = n4 - 4 - 4 * qq, d1 = n2 - 4 - 4 * qq;
        const int ka = tb.bitrev[2 * qq], kb = tb.bitrev[2 * qq + 1];
        float a[NP][4], b[NP][4];
#pragma unroll
        for (int q = 0; q < NP; q++) {
            const float *Uq = U + q * bs;
#pragma unroll
            for (int k = 0; k < 4; k++) { a[q][k] = Uq[ka + k]; b[q][k] = Uq[kb + k]; }
        }
#pragma unroll
        for (int q = 0; q < NP; q++) {
            float *Vq = V + q * bs;
            Vq[d1 + 3] = a[q][0]; Vq[d1 + 2] = a[q][1]; Vq[d0 + 3] = a[q][2]; Vq[d0 + 2] = a[q][3];
            Vq[d1 + 1] = b[q][0]; Vq[d1 + 0] = b[q][1]; Vq[d0 + 1] = b[q][2]; Vq[d0 + 0] = b[q][3];
        }
    }
    sync();
    // step 7 (imdct.rs:533-580), in place on V
    for (int t = tid; t < (n >> 4); t += NT) {
        const int d = 4 * t, e = n2 - 4 - 4 * t, co = 4 * t;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int dd = d + 2 * h, ee = e + 2 - 2 * h;
            const float c0 = Cc[co + 2 * h], c1 = Cc[co + 2 * h + 1];
            float vd[NP], vd1[NP], ve[NP], ve1[NP];
#pragma unroll
            for (int q = 0; q < NP; q++) {
                const float *Vq = V + q * bs;
                vd[q] = Vq[dd]; vd1[q] = Vq[dd + 1]; ve[q] = Vq[ee]; ve1[q] = Vq[ee + 1];
            }
#pragma unroll
            for (int q = 0; q < NP; q++) {
                float *Vq = V + q * bs;
                const float a02 = __fsub_rn(vd[q], ve[q]);
                const float a11 = __fadd_rn(vd1[q], ve1[q]);
                const float b0 = __fadd_rn(__fmul_rn(c1, a02), __fmul_rn(c0, a11));
                const float b1 = __fsub_rn(__fmul_rn(c1, a11), __fmul_rn(c0, a02));
                const float b2 = __fadd_rn(vd[q], ve[q]);
                const float b3 = __fsub_rn(vd1[q], ve1[q]);
                Vq[dd] = __fadd_rn(b2, b0);
                Vq[dd + 1] = __fadd_rn(b3, b1);
                Vq[ee] = __fsub_rn(b2, b0);
                Vq[ee + 1] = __fsub_rn(b1, b3);
            }
        }
    }
    sync();
}

// Step 8 of inverse_mdct (imdct.rs:589-658) for output index m < n/4, from the post-step-7 buffer V: (p_odd, p_even),
// which give x[m] = p_odd, x[n2-1-m] = -p_odd, x[n2+m] = p_even, x[n-1-m] = p_even.
__device__ __forceinline__ float2 d_imdct_step8(const float *V, const float *__restrict__ B, int n2, int m)
{
    const int ee = n2 - 2 - 2 * m;                // V/B pair consumed for output index m
    const float v0 = V[ee], v1 = V[ee + 1];
    const float b0 = __ldg(B + ee), b1 = __ldg(B + ee + 1);
    return make_float2(__fsub_rn(__fmul_rn(v0, b1), __fmul_rn(v1, b0)), __fsub_rn(__fmul_rn(-v0, b0), __fmul_rn(v1, b1)));
}

// grid = (packets, max channels); dynamic smem = n floats (U and V halves).
// in: spectrum [channels][n/2] at coeff_off; out: x [channels][n] at x_off.
__global__ void __launch_bounds__(kImdctThreads)
k_imdct(const DevPacket *__restrict__ pkts, const float *__restrict__ spec, float *__restrict__ xout)
{
    const DevPacket &p = pkts[blockIdx.x];
    const int ch = blockIdx.y;
    if (ch >= p.channels) return;
    const DevTables &tb = p.setup->tab[p.blockflag];
    const int n = p.n, n2 = n >> 1, n4 = n >> 2;
    const float *__restrict__ B = tb.b;
    const float *__restrict__ X = spec + p.coeff_off + (size_t)ch * n2;
    float *__restrict__ out = xout + p.x_off + (size_t)ch * n;
    extern __shared__ float smem[];
    float *U = smem, *V = smem + n2;
    const int tid = threadIdx.x;
    d_imdct_to_v<1>(tb, n, X, 0, U, V, 0, tid, kImdctThreads, [] { __syncthreads(); });
    for (int m = tid; m < n4; m += kImdctThreads) {
        const float2 pp = d_imdct_step8(V, B, n2, m);
        out[m] = pp.x;
        out[n2 - 1 - m] = -pp.x;
        out[n2 + m] = pp.y;
        out[n - 1 - m] = pp.y;
    }
}

// ---------------------------------------------------------------------------------------------
// window / overlap-add / slice / sample conversion, audio.rs:1079-1157 + samples.rs
// ---------------------------------------------------------------------------------------------
// the sample conversions (samples.rs:86-103, and f16) and store_sample live in kernel_long.cuh, shared by every path

constexpr int kOverlapThreads = 256;

// Output channel k of the setup's mix (lwb_setup_set_output_mix) at one sample; x(c) gives input channel c's f32 sample.
// The rounded products are summed left to right in ascending channel order, the first one not added to a zero; a row
// without terms gives +0.0f.
template <class X>
__device__ __forceinline__ float d_mix_sample(const DevSetup &su, int k, X x)
{
    const int a = su.mix_row[k], b = su.mix_row[k + 1];
    if (a == b) return 0.f;
    float y = __fmul_rn(__ldg(su.mix_w + a), x(su.mix_ch[a]));
    for (int j = a + 1; j < b; j++) y = __fadd_rn(y, __fmul_rn(__ldg(su.mix_w + j), x(su.mix_ch[j])));
    return y;
}

// Sample i < plen of a block's left part, x, overlap-added with sample i of the previous block's right half, pv
// (audio.rs:1116-1118): x windowed by w, pv by w in reverse, summed.  Samples from plen on pass unchanged.
__device__ __forceinline__ float d_overlap_add(float x, float pv, const float *__restrict__ w, int plen, int i)
{
    return __fadd_rn(__fmul_rn(x, w[i]), __fmul_rn(pv, w[plen - 1 - i]));
}

// grid.y is the output channel k of the packet's setup: its input channel without MIX or without a mix.  MIX: each block
// recomputes the overlap-add of the input channels row k uses, from x and the previous right half, and stores their mix.
template <int FORMAT, bool MIX = false>
__global__ void __launch_bounds__(kOverlapThreads)
k_overlap(const DevPacket *__restrict__ pkts, const float *__restrict__ x, void *__restrict__ pcm)
{
    const DevPacket &p = pkts[blockIdx.x];
    const DevSetup &su = *p.setup;
    const int ch = blockIdx.y;
    const bool mix = MIX && su.n_out;
    const int K = mix ? su.n_out : p.channels;
    if (ch >= K || p.plen == 0) return;                // audio.rs:1140-1151: no previous -> no output
    const int n = p.n, plen = p.plen, ls = p.ls, olen = p.rs - p.ls;
    const float *__restrict__ w = su.tab[p.slope_sel].window;
    const DevPacket *q = p.prev_packet >= 0 ? &pkts[p.prev_packet] : nullptr;
    auto prev_of = [&](int c) {                        // channel c's previous right half
        return q ? x + q->x_off + (size_t)c * q->n + p.prev_rs : p.state + (size_t)c * p.state_stride;
    };
    const float *__restrict__ prev_ch = prev_of(ch);   // without MIX, every sample's channel is ch
    for (int i = threadIdx.x; i < olen; i += kOverlapThreads) {
        auto ola = [&](int c) {                        // the unmixed sample of channel c
            const float v = x[p.x_off + (size_t)c * n + ls + i];
            return i < plen ? d_overlap_add(v, (MIX ? prev_of(c) : prev_ch)[i], w, plen, i) : v;
        };
        store_sample<FORMAT>(pcm, p.out_off, p.out_stride, K, ch, i, mix ? d_mix_sample(su, ch, ola) : ola(ch));
    }
}

// grid = (packets, max channels): packets flagged save_state copy x[rs..re) into the stream state.
__global__ void __launch_bounds__(kOverlapThreads)
k_save_state(const DevPacket *__restrict__ pkts, const float *__restrict__ x)
{
    const DevPacket &p = pkts[blockIdx.x];
    const int ch = blockIdx.y;
    if (!p.save_state || ch >= p.channels) return;
    const float *__restrict__ xc = x + p.x_off + (size_t)ch * p.n + p.rs;
    float *__restrict__ st = p.state + (size_t)ch * p.state_stride;
    for (int i = threadIdx.x; i < p.re - p.rs; i += kOverlapThreads) st[i] = xc[i];
}

}  // namespace lwb
