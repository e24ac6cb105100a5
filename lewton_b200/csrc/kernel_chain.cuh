// kernel_chain.cuh -- the general synthesis kernel: any blocksize 6..13, mixed short/long
// sequences, up to 8 channels, spectrum, residue or VQ entry, all output formats, in ONE launch.
//
// One CTA owns one chain (consecutive packets of one stream), one group of `wpc` warps per channel
// (1 warp for small blocks, up to 8 for n = 8192; the group synchronises on its own named barrier).
// The group keeps its channel's working buffers (U, V: n/2 floats each) and the previous block's right half
// (PreviousWindowRight, audio.rs:847-861) in shared memory for the whole chain, so HBM sees only the
// algorithmic traffic: coefficients in, PCM out, the stream state once per chain.  Per packet:
//   VQ entry:      the whole CTA accumulates the packet's residue vectors from its VQ records into a [C][n/2]
//                  region of shared memory (d_vq_accumulate, kernel_prologue.cuh), then goes on as the residue
//                  entry does, reading them there instead of from the coefficient arena;
//   residue entry: floor-1 posts per channel (one lane, serial, <= 65 posts; floor-0 curves come rendered by
//                  k_floor0_curves) -> the whole CTA does
//                  inverse coupling + floor x residue bin-parallel straight into the channels'
//                  shared buffers (audio.rs:991-1039);
//   every warp:    inverse MDCT stage by stage in shared memory (imdct.rs:291-659, literal schedule),
//                  window / overlap-add / slice / sample conversion (audio.rs:1056-1157) with step 8
//                  evaluated on the fly per output sample.
// Window geometry (audio.rs:1056-1073) is recomputed on the device from the three mode bytes of a
// packet; the host has already walked the chain once to catch the OLA guard and size the output.
//
// This is the fallback for everything the fused long-block kernel (kernel_long.cuh) does not take;
// it replaces the four-kernel path (kernels_generic.cuh) wherever channels <= 8 and the buffers fit
// in shared memory: a chain's buffers and state stay there instead of round-tripping HBM between kernels.
#pragma once
#include "kernels_generic.cuh"
#include "kernel_prologue.cuh"

namespace lwb {

struct ChainDesc {
    const DevSetup *setup;
    float *state;              // [channels][state_stride]
    uint64_t coeff_off;        // first packet's [channels][n/2] in the coefficient arena
    uint64_t out_off;          // chain's first PCM element
    uint64_t out_stride;       // planar: elements between channel planes
    uint64_t pkt_index;        // first row in the per-packet floor arenas
    uint32_t n_packets;
    uint32_t byte_off;         // offset of this chain's (mode, prev, next) triples
    uint32_t state_stride;
    uint16_t plen0;            // length of the stream's saved right half when the chain starts
    uint8_t has0;              // 1 if the stream has history
    uint8_t channels;
};

// x[j] of the IMDCT output, from the post-step-7 buffer V: the one step-8 product (d_imdct_step8) that gives it
__device__ __forceinline__ float d_x_at(const float *V, const float *__restrict__ B, int n, int j)
{
    const int n2 = n >> 1, n4 = n >> 2;
    if (j < n2) {
        const bool mir = j >= n4;
        const float p_odd = d_imdct_step8(V, B, n2, mir ? n2 - 1 - j : j).x;
        return mir ? -p_odd : p_odd;
    }
    const int jj = j - n2;
    return d_imdct_step8(V, B, n2, jj >= n4 ? n2 - 1 - jj : jj).y;
}

// MULTI = false: one warp per channel (<= 8 warps, compile-time group size, warp-level syncs);
// MULTI = true: `wpc` warps per channel, named barriers.
// np: blocks a channel group transforms together (spectrum entry, !MULTI; the host sizes shared memory for it).
// vq: the batch's VQ arrays (VQ entry; `coeffs` is not read then).
// MIX: the chain's setup may have an output mix (lwb_setup_set_output_mix).  The channel groups then write their
// overlap-added samples into a [C][n1max/2] tile -- each group's U half of the block, free once its transform is done --
// and after a CTA barrier the whole CTA forms the K output channels from it and stores them; a setup without a mix has
// K = C and copies its channels.  Every group, active or not, reaches the barriers (olen is the same for every channel).
template <int FORMAT, int ENTRY, bool MULTI, bool MIX = false>
__global__ void __launch_bounds__(MULTI ? 1024 : 256)
k_chain(const ChainDesc *__restrict__ chains, const uint8_t *__restrict__ pkt_bytes, const float *__restrict__ coeffs,
        const float *__restrict__ dense_floor, const uint8_t *__restrict__ floor_kind,
        const uint32_t *__restrict__ floor1_y, void *__restrict__ pcm, int n1max, int wpc, int np,
        const float *__restrict__ zero_floor, VqDev vq)
{
    extern __shared__ float ch_smem[];
    const ChainDesc cd = chains[blockIdx.x];
    const DevSetup &su = *cd.setup;
    const int C = cd.channels;
    const int gt = MULTI ? wpc * 32 : 32;                      // threads per channel group
    const int warp = threadIdx.x / gt, lane = threadIdx.x % gt, W = blockDim.x / gt;   // "warp" = channel group
    const bool active = warp < C;
    auto gsync = [&]() {
        if (!MULTI) __syncwarp();
        else asm volatile("bar.sync %0, %1;" ::"r"(warp + 1), "r"(gt) : "memory");
    };
    // per channel group: `np` blocks of U | V (n1max floats each), then the previous right half
    const int per_warp = np * n1max + (n1max >> 1);
    float *U = ch_smem + (size_t)warp * per_warp, *prev = U + np * n1max;
    // floor posts of up to 8 channels (residue entry)
    uint16_t *s_x = reinterpret_cast<uint16_t *>(ch_smem + (size_t)W * per_warp);
    uint16_t *s_y = s_x + 8 * (LWB_MAX_POSTS + 1);
    int *s_m = reinterpret_cast<int *>(s_y + 8 * (LWB_MAX_POSTS + 1));
    // VQ entry: the packet's residue vectors, [C][n/2] (the host sizes this region for C * n1max / 2 floats)
    float *s_acc = reinterpret_cast<float *>(s_m + 8);

    const int n0 = 1 << su.bs0;
    bool has = cd.has0;
    int plen = cd.plen0;
    if (active && has)
        for (int i = lane; i < plen; i += gt) prev[i] = cd.state[(size_t)warp * cd.state_stride + i];
    uint64_t coeff = cd.coeff_off;
    uint64_t pos = 0;                     // samples per channel emitted so far
    const uint8_t *bytes = pkt_bytes + cd.byte_off;

    for (uint32_t p = 0; p < cd.n_packets;) {
        const int blockflag = su.mode_blockflag[bytes[3 * p]];
        const DevTables &tb = su.tab[blockflag];
        const int n = 1 << tb.bs, n2 = n >> 1;
        // consecutive packets of one blocksize are transformed together (they are independent until the
        // overlap-add): up to `np` blocks in flight per channel group
        uint32_t g = 1;
        if (ENTRY == LWB_ENTRY_SPECTRUM && !MULTI)
            while (g < (uint32_t)np && p + g < cd.n_packets && su.mode_blockflag[bytes[3 * (p + g)]] == blockflag) g++;

        if (ENTRY != LWB_ENTRY_SPECTRUM) {
            const int mode = bytes[3 * p];
            const DevMapping &mp = su.mappings[su.mode_mapping[mode]];
            const uint64_t row = (cd.pkt_index + p) * C;
            __syncthreads();              // previous packet finished with U/V, the post arrays and the accumulators
            if (active && lane == 0 && floor_kind[row + warp] == LWB_FLOOR_ONE) {
                const DevFloor1 &fl = su.floors[mp.floor_of_channel[warp]];
                s_m[warp] = d_floor1_posts(fl, floor1_y + (row + warp) * LWB_MAX_POSTS, n2,
                                           s_x + warp * (LWB_MAX_POSTS + 1), s_y + warp * (LWB_MAX_POSTS + 1));
            }
            if (ENTRY == LWB_ENTRY_VQ) {
                const uint64_t pk = cd.pkt_index + p;
                const uint64_t o0 = vq.run_off[pk], e0 = vq.ent_off[pk];
                d_vq_accumulate(s_acc, C, n2, su, mp, vq.runs + o0, (uint32_t)(vq.run_off[pk + 1] - o0), vq.entries + e0,
                                (uint32_t)(vq.ent_off[pk + 1] - e0), threadIdx.x, blockDim.x);
            }
            __syncthreads();
            const int nsteps = mp.n_coupling;
            for (int k = threadIdx.x; k < n2; k += blockDim.x) {
                float r[8];
#pragma unroll
                for (int c = 0; c < 8; c++)
                    r[c] = c < C ? (ENTRY == LWB_ENTRY_VQ ? s_acc[c * n2 + k] : coeffs[coeff + (size_t)c * n2 + k]) : 0.f;
                d_inverse_couple_regs(r, mp, nsteps);
#pragma unroll
                for (int c = 0; c < 8; c++) {
                    if (c < C) {
                        const int kind = floor_kind[row + c];
                        const float f = kind == LWB_FLOOR_ONE
                                            ? c_inverse_db[d_floor1_y_at(s_x + c * (LWB_MAX_POSTS + 1), s_y + c * (LWB_MAX_POSTS + 1),
                                                                         s_m[c], k) & 255u]
                                            : d_floor_other(kind, dense_floor, zero_floor, coeff + (size_t)c * n2 + k);
                        ch_smem[(size_t)c * per_warp + k] = __fmul_rn(f, r[c]);      // channel c's U
                    }
                }
            }
            __syncthreads();
        }

        if (active) {
            float *V0 = U + (n1max >> 1);
            if (ENTRY != LWB_ENTRY_SPECTRUM) {
                d_imdct_to_v<1>(tb, n, U, 0, U, V0, 0, lane, gt, gsync);
            } else {
                const float *X = coeffs + coeff + (size_t)warp * n2;
                const size_t xs = (size_t)C * n2;
                uint32_t q = 0;
                while (q < g) {                                  // pieces of 4, 2, 1 blocks
                    const uint32_t rem = g - q;
                    if (rem >= 4) { d_imdct_to_v<4>(tb, n, X + q * xs, xs, U + q * n1max, V0 + q * n1max, n1max, lane, gt, gsync); q += 4; }
                    else if (rem >= 2) { d_imdct_to_v<2>(tb, n, X + q * xs, xs, U + q * n1max, V0 + q * n1max, n1max, lane, gt, gsync); q += 2; }
                    else { d_imdct_to_v<1>(tb, n, X + q * xs, xs, U + q * n1max, V0 + q * n1max, n1max, lane, gt, gsync); q += 1; }
                }
            }
        }
        for (uint32_t q = 0; q < g; q++) {
            const bool pf = blockflag ? bytes[3 * (p + q) + 1] != 0 : true;       // short blocks: map_or(true, ..)
            const bool nf = blockflag ? bytes[3 * (p + q) + 2] != 0 : true;
            // audio.rs:1056-1073
            const int ls = pf ? 0 : (n - n0) >> 2;
            const int slope_sel = pf ? blockflag : 0;
            const int rs = nf ? n2 : (n * 3 - n0) >> 2;
            const int re = nf ? n : (n * 3 + n0) >> 2;
            const int olen = rs - ls;
            const float *V = U + q * n1max + (n1max >> 1);
            const float *__restrict__ B = tb.b;
            if (has) {
                const float *__restrict__ w = su.tab[slope_sel].window;
                if constexpr (MIX) {
                    constexpr bool planar = out_format_of(FORMAT).planar;
                    const int T = n1max >> 1, K = su.n_out ? su.n_out : C;
                    for (int t0 = 0; t0 < olen; t0 += T) {
                        const int tn = min(T, olen - t0);
                        if (active)
                            for (int i = lane; i < tn; i += gt) {
                                const int j = t0 + i;
                                float v = d_x_at(V, B, n, ls + j);
                                if (j < plen) v = d_overlap_add(v, prev[j], w, plen, j);
                                U[q * n1max + i] = v;
                            }
                        __syncthreads();
                        for (int e = threadIdx.x; e < K * tn; e += blockDim.x) {
                            const int k = planar ? e / tn : e % K, t = planar ? e % tn : e / K;
                            auto x = [&](int c) { return ch_smem[(size_t)c * per_warp + q * n1max + t]; };
                            store_sample<FORMAT>(pcm, cd.out_off, cd.out_stride, K, k, pos + t0 + t, su.n_out ? d_mix_sample(su, k, x) : x(k));
                        }
                        __syncthreads();
                    }
                } else if (active) {
                    for (int i = lane; i < olen; i += gt) {
                        float v = d_x_at(V, B, n, ls + i);
                        if (i < plen) v = d_overlap_add(v, prev[i], w, plen, i);
                        store_sample<FORMAT>(pcm, cd.out_off, cd.out_stride, C, warp, pos + i, v);
                    }
                    gsync();                                   // every lane has read prev before it is refilled
                }
            }
            plen = re - rs;                                    // audio.rs:1121
            if (active) {
                for (int i = lane; i < plen; i += gt) prev[i] = d_x_at(V, B, n, rs + i);
                gsync();
            }
            if (has) pos += olen;
            has = true;
            coeff += (uint64_t)C * n2;
        }
        p += g;
    }
    if (active)
        for (int i = lane; i < plen; i += gt) cd.state[(size_t)warp * cd.state_stride + i] = prev[i];
}

}  // namespace lwb
