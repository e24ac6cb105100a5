// kernel_mid.cuh -- fused IMDCT + window + overlap-add for runs of blocks of n = 1024 and n = 512 (blocksizes 10 and 9):
// the register-resident structure of kernel_long.cuh for the 8- and 7-bit index spaces (below: n = 1024; n = 512 has two
// block bits, four runs per warp, step 2 alone in phase A and stages 0, 1, 2 in phase B).
//
// A 1024-point block has 256 complex values; a warp holds 512, so it transforms TWO blocks in lockstep -- two different
// runs of equal length, like k_short_g's positions.  The block index is made the TOP bit of kernel_long's 9-bit element
// index, c = 256 blk + c', which leaves every index map, both transposes and their swizzle exactly as they are:
//     phase A: slot = (blk, c'7, c'6)   step 0, step 2 (bit 7: slots j, j + 2), stage 0 (bit 6: slots j, j + 1)
//     phase B: slot = c'5 c'4 c'3       stages 1, 2, 3 -- kernel_long's phase_b, other twiddles
//     phase C: slot = c'2 c'1 c'0       ld654, renaming, step 7, step 8, window / OLA -- kernel_long's phase_c_fft
// with one change to the phase-C map: kernel_long's second half of a lane holds the element whose upper six bits are
// complemented (the step-7 partner, imdct.rs:533-580); complementing the block bit as well would pair the two blocks, so
// here only the five bits inside the block are complemented (elemC_m).  A lane then carries elements of block
// (lane & 1) only in phase C, its output samples are m = 32 rev3(slot) + (lane >> 1) and the mirror images, and the
// overlap state of "its" run stays in its registers from packet to packet.
//
// The lane functions compile for the host too: tests/emu/mid_emu.cpp runs the 32 lanes sequentially against the oracle.
#pragma once
#include "kernel_long.cuh"

namespace lwb {

// KB = number of block bits: 1 -> n = 1024 (two runs per warp), 2 -> n = 512 (four runs per warp)
template <int KB>
struct Mid {
    static_assert(KB == 1 || KB == 2, "k_mid covers n = 1024 and n = 512");
    static constexpr int NB = 1 << KB;            // runs (blocks) per warp
    static constexpr int BS = 11 - KB;            // blocksize (log2 n)
    static constexpr int N = 2048 >> KB;
    static constexpr int N2 = 1024 >> KB;         // spectrum floats / PCM samples per block
    static constexpr int C = 512 >> KB;           // complex elements per block
    static constexpr int K = 9 - KB;              // index bits per block
    static constexpr int SPB = 8 >> KB;           // phase-A slots per block
    static constexpr int W = 64 >> KB;            // output samples per (slot, half-row)
    static constexpr int TMASK = (1 << (6 - KB)) - 1;   // the bits of T inside the block
};
constexpr int kMidBs = 10;                        // (KB = 1)

// phase C: the element of (lane, slot, half): upper bits T = (blk, T'), half 1 complements T' only
template <int KB>
LWB_HD int elemC_m(int lane, int slot, int half)
{
    const int T0 = rev6(lane);
    return 8 * (half ? (T0 ^ Mid<KB>::TMASK) : T0) + slot;
}
// block of a lane in phase C (the top KB bits of T = the low KB bits of the lane, reversed), and the output index m
// (0 .. C - 1) of (lane, slot, half) AFTER the step-7 half swap
template <int KB>
LWB_HD int blockC_m(int lane) { return KB == 1 ? (lane & 1) : (((lane & 1) << 1) | ((lane >> 1) & 1)); }
template <int KB>
LWB_HD int outIndex_m(int lane, int slot, int half)
{
    const int flip = (slot & 1) ? half : !half;
    return Mid<KB>::W * rev3(slot) + (flip ? Mid<KB>::W - 1 - (lane >> KB) : (lane >> KB));
}
template <int KB>
LWB_HD int revK_m(int c) { return rev9(c & (Mid<KB>::C - 1)) >> KB; }          // bit reversal of K bits

// Host: per-lane pack from the blocksize-(11 - KB) tables (a, b: n/2; c: n/4; w: n/2).  Same slot layout as
// long_build_pack; P_S2W* uses entries 0 .. SPB/2 - 1, P_L0W* entry 0 (KB = 1 only), P_L1W* is unused; P_L2 / P_L3 / P_L4
// carry the three stages of phase B (stages K-7, K-6, K-5).
template <int KB>
inline void mid_build_pack(const float *a, const float *b, const float *c, const float *w, float *pack)
{
    using M = Mid<KB>;
    V *P = reinterpret_cast<V *>(pack);
    for (int i = 0; i < P_END * 32; i++) P[i] = V{0.f, 0.f};
    for (int lane = 0; lane < 32; lane++) {
        auto put = [&](int slot, float x, float y) { P[slot * 32 + lane] = V{x, y}; };
        float tx[2], ty[2];
        // phase A: c' = elemA & (C - 1)
        for (int j = 0; j < 8; j++) {                          // step 0 (imdct.rs:337-371)
            for (int h = 0; h < 2; h++) {
                const int cc = elemA(lane, j, h) & (M::C - 1);
                const float s = cc < M::C / 2 ? -1.0f : 1.0f;  // (-x)*A == x*(-A)
                tx[h] = s * a[M::N2 - 2 - 2 * cc];
                ty[h] = s * a[M::N2 - 1 - 2 * cc];
            }
            put(P_S0W0 + j, tx[0], tx[1]);
            put(P_S0W1 + j, ty[0], ty[1]);
        }
        for (int u = 0; u < M::SPB / 2; u++) {                 // step 2 (imdct.rs:385-430): lower element (top bit 0), slot u
            for (int h = 0; h < 2; h++) {
                const int cc = elemA(lane, u, h) & (M::C - 1);
                tx[h] = a[M::N2 - 4 - 4 * cc];
                ty[h] = a[M::N2 - 3 - 4 * cc];
            }
            put(P_S2W0 + u, tx[0], tx[1]);
            put(P_S2W1 + u, ty[0], ty[1]);
        }
        if (KB == 1) {                                         // stage 0 on bit 6: a = r * 8
            for (int h = 0; h < 2; h++) {
                const int r = (~elemA(lane, 1, h)) & 63;
                tx[h] = a[8 * r];
                ty[h] = a[8 * r + 1];
            }
            put(P_L0W0, tx[0], tx[1]);
            put(P_L0W1, ty[0], ty[1]);
        }
        // phase B: bits 5, 4, 3 = stages K-7, K-6, K-5 (a = r * (8 << stage)); both halves share the twiddle
        const int k5 = 8 << (M::K - 7), k4 = 8 << (M::K - 6), k3 = 8 << (M::K - 5);
        for (int u = 0; u < 4; u++) {
            const int r = (~elemB(lane, 4 + u, 0)) & 31;
            put(P_L2W0 + u, a[k5 * r], a[k5 * r]);
            put(P_L2W1 + u, a[k5 * r + 1], a[k5 * r + 1]);
        }
        for (int u = 0; u < 2; u++) {
            const int r = (~elemB(lane, 2 + u, 0)) & 15;
            put(P_L3W0 + u, a[k4 * r], a[k4 * r]);
            put(P_L3W1 + u, a[k4 * r + 1], a[k4 * r + 1]);
        }
        {
            const int r = (~elemB(lane, 1, 0)) & 7;
            put(P_L4W0, a[k3 * r], a[k3 * r]);
            put(P_L4W1, a[k3 * r + 1], a[k3 * r + 1]);
        }
        // phase C
        put(P_A2, a[M::N >> 3], a[M::N >> 3]);
        for (int jj = 0; jj < 4; jj++) {
            for (int h = 0; h < 2; h++) {
                const int p = M::C - 1 - revK_m<KB>(elemC_m<KB>(lane, 2 * jj + 1, h));     // step-7 index of the D side
                tx[h] = c[2 * p];
                ty[h] = c[2 * p + 1];
            }
            put(P_S7C0 + jj, tx[0], tx[1]);
            put(P_S7C1 + jj, ty[0], ty[1]);
        }
        for (int j = 0; j < 8; j++) {
            float b0[2], b1[2], wl[2], wh[2];
            for (int h = 0; h < 2; h++) {
                const int m = outIndex_m<KB>(lane, j, h);
                const int cp = M::C - 1 - m;                   // V element feeding output m
                b0[h] = b[2 * cp];
                b1[h] = b[2 * cp + 1];
                wl[h] = w[m];
                wh[h] = w[M::N2 - 1 - m];
            }
            put(P_B0 + j, b0[0], b0[1]);
            put(P_B1 + j, b1[0], b1[1]);
            put(P_WLO + j, wl[0], wl[1]);
            put(P_WHI + j, wh[0], wh[1]);
        }
    }
}

// Phase A.  tile[blk] = the block's n/2 spectrum floats.  Quad #f (4 floats at 4f) yields element c' = f from (q1, q3) and
// c' = C - 1 - f from (q0, q2) (step 0, imdct.rs:337-371).  The lane reads quads #(lane + 64 m) and #(63 - lane + 64 m),
// m < SPB / 2, of every block: they feed slots m and SPB - 1 - m of the block's SPB.
template <int KB, class TW>
LWB_HD void phase_a_m(const float *const tile[], int lane, TW tw, V O[8], V E[8])
{
    using M = Mid<KB>;
#pragma unroll
    for (int blk = 0; blk < M::NB; blk++)
#pragma unroll
        for (int m = 0; m < M::SPB / 2; m++) {
            const Q4 f1 = ld_q4(tile[blk] + 4 * (lane + 64 * m));
            const Q4 f2 = ld_q4(tile[blk] + 4 * (63 - lane + 64 * m));
            {
                const int j = M::SPB * blk + m;
                const V w0 = tw(P_S0W0 + j), w1 = tw(P_S0W1 + j);
                const V qa = V{f1.w, f2.w}, qb = V{f1.y, f2.y};
                O[j] = vsub_p(vmul(qa, w0), vmul(qb, w1));
                E[j] = vadd_p(vmul(qa, w1), vmul(qb, w0));
            }
            {
                const int j = M::SPB * blk + M::SPB - 1 - m;
                const V w0 = tw(P_S0W0 + j), w1 = tw(P_S0W1 + j);
                const V qa = V{f2.x, f1.x}, qb = V{f2.z, f1.z};
                O[j] = vsub_p(vmul(qa, w0), vmul(qb, w1));
                E[j] = vadd_p(vmul(qa, w1), vmul(qb, w0));
            }
        }
    // step 2 (imdct.rs:385-430): the top bit of c' = slot bit 2 - KB
#pragma unroll
    for (int blk = 0; blk < M::NB; blk++)
#pragma unroll
        for (int u = 0; u < M::SPB / 2; u++) {
            const int j = M::SPB * blk + u;
            bfly(O[j + M::SPB / 2], E[j + M::SPB / 2], O[j], E[j], tw(P_S2W0 + u), tw(P_S2W1 + u));
        }
    if (KB == 1) {          // stage 0 (imdct.rs:445-446): bit 6 = slot bit 0
        const V w0 = tw(P_L0W0), w1 = tw(P_L0W1);
#pragma unroll
        for (int j = 1; j < 8; j += 2) bfly(O[j], E[j], O[j - 1], E[j - 1], w0, w1);
    }
}

#if defined(__CUDACC__)
// ---------------------------------------------------------------------------------------------
// device side: k_mid<OutT, KB>.  Descriptors: groups of NB = 2^KB LongRun (48 B each; in_stride / out in N2-sample units of
// this blocksize, first_short / last_short unused) of equal n_packets -- the host pads a short group with dummies --,
// under kernel_deal.cuh's static-deal driver: one group per item, one packet per unit (a stage = the runs' tiles, 4 KB
// together, which then serve as the E | O planes of the transposes), and the state rows of a group with history.
// ---------------------------------------------------------------------------------------------
constexpr int kMidFetch = 3;
template <int KB>
struct MidDev {           // n = 512: four descriptors per group -- one ring stage less keeps the CTA inside 227 KB
    static constexpr int Ring = KB == 1 ? kLongRing : kLongRing - 1;
    static constexpr int Slots = kMidFetch + Ring + 3;
    static constexpr size_t Smem = 2048 + (size_t)kLongWarps * (Ring + 1) * kLongTileBytes + (size_t)kLongPackFloats * 4 +
                                   kLongWarps * (Ring + 2) * 8 + (size_t)kLongWarps * Slots * Mid<KB>::NB * sizeof(LongRun) + 64;
};

template <typename OutT, int KB>
__global__ void __launch_bounds__(kLongWarps * 32, 1)
k_mid(const LongRun *__restrict__ runs, uint32_t n_groups, const float *__restrict__ pack)
{
    using M = Mid<KB>;
    constexpr int NB = M::NB;
    constexpr uint32_t kTile = M::N2 * 4;                      // bytes of one run's tile / state row
    constexpr uint32_t kGroupBytes = NB * sizeof(LongRun);
    constexpr int kRing = MidDev<KB>::Ring, kSlots = MidDev<KB>::Slots;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int blk = blockC_m<KB>(lane);                        // the run of the group whose samples this lane ends up with
    const LongSmem<kRing, kLongTileBytes, kSlots * NB> sm(smem_raw, warp);
    const float *tiles = sm.tiles, *s_state = sm.s_state;     // s_state: [NB][N2]
    LongRun *s_desc = sm.s_desc;
    V twR[kTwRegs];
    long_cta_setup(pack, sm.s_pack, sm.bars, kRing + 1, lane, twR);
    const TwMix tw{twR, sm.s_pack + lane};

    const uint32_t state_s = smem_u32(s_state);
    const uint32_t lA0 = laneA(lane, 0), lA1 = laneA(lane, 1);
    const uint32_t lB = laneB(lane);
    const uint32_t lC0 = 4u * (uint32_t)swz(elemC_m<KB>(lane, 0, 0)), lC1 = 4u * (uint32_t)swz(elemC_m<KB>(lane, 0, 1));

    const uint32_t W = gridDim.x * kLongWarps, gw = blockIdx.x * kLongWarps + warp;
    if (gw >= n_groups) return;
    StaticDeal<kGroupBytes / 16, kSlots, kMidFetch, kRing, kLongTileBytes> deal(
        runs, n_groups, W, gw, smem_u32(s_desc), smem_u32(tiles), smem_u32(sm.bars), lane);
    auto units = [&](uint32_t sl) { return s_desc[NB * sl].n_packets; };
    auto issue = [&](uint32_t sl, uint32_t pkt, uint32_t bar, uint32_t dst) {     // lanes b < NB issue run b's tile
        if (lane == 0) mbar_expect_tx(bar, NB * kTile);
        __syncwarp();
        if (lane < NB) {
            const LongRun &r = s_desc[NB * sl + lane];
            fence_proxy_async();          // the stage was written through the generic proxy (transposes) before
            tma_load_1d(dst + lane * kTile, r.in + (size_t)pkt * r.in_stride, kTile, bar);
        }
    };
    auto group_has_state = [&](uint32_t sl) {
        bool any = false;
#pragma unroll
        for (int b = 0; b < NB; b++) any |= s_desc[NB * sl + b].has_prev != 0;
        return any;
    };
    auto issue_state = [&](uint32_t sl, uint32_t bar) {        // lanes b < NB with history issue their row
        const bool mine = lane < NB && s_desc[NB * sl + (lane < NB ? lane : 0)].has_prev != 0;
        const uint32_t n = (uint32_t)__popc(__ballot_sync(0xffffffffu, mine));
        if (lane == 0) mbar_expect_tx(bar, n * kTile);
        __syncwarp();
        if (mine) {
            fence_proxy_async();
            tma_load_1d(state_s + lane * kTile, s_desc[NB * sl + lane].state, kTile, bar);
        }
    };
    deal.start(units, issue);

    for (uint32_t c_grp = gw; c_grp < n_groups; c_grp += W) {
        const uint32_t my_slot = deal.take_slot();
        const LongRun *g = s_desc + NB * my_slot;
        const uint32_t npk = g[0].n_packets;
        const bool grp_state = group_has_state(my_slot);
        // this lane's run (the descriptor slot of the group being consumed is never the target of a fetch)
        const LongRun &mr = g[blk];
        const uint32_t flags = (mr.has_prev ? 1u : 0u) | (mr.write_state ? 2u : 0u) | (mr.dummy ? 4u : 0u);
        OutT *out = static_cast<OutT *>(mr.out);
        float *state_g = mr.state;
        deal.begin_state(c_grp, group_has_state, issue_state);
        V pe[8];
#pragma unroll
        for (int j = 0; j < 8; j++) pe[j] = V{0.f, 0.f};

        for (uint32_t p = 0; p < npk; p++) {
            const uint32_t stage = deal.wait_stage();
            V O[1][8], E[1][8];
            {
                const float *tp[NB];
#pragma unroll
                for (int b = 0; b < NB; b++) tp[b] = tiles + stage * kLongN2 + b * M::N2;
                phase_a_m<KB>(tp, lane, tw, O[0], E[0]);
            }
            transpose_abc<1>(tw, deal.ring_s + stage * kLongTileBytes, lA0, lA1, lB, lC0, lC1, O, E);
            deal.produce(units, issue);             // the stage is free again
            phase_c_fft<1>(tw, O, E);
            if (p > 0) {
                out_block<M::W, M::N2 - M::W, false>(tw, lane >> KB, O[0], E[0], pe, flags, out, s_state + blk * M::N2);
            } else {
                if (grp_state) deal.wait_state(c_grp, issue_state);
                out_block<M::W, M::N2 - M::W, true>(tw, lane >> KB, O[0], E[0], pe, flags, out, s_state + blk * M::N2);
                __syncwarp();
                if (grp_state) deal.release_state(c_grp, group_has_state, issue_state);   // state tile consumed
            }
            if (p > 0 || (flags & 1u)) out += M::N2;
            deal.next_stage();
        }
        if ((flags & 6u) == 2u)               // write_state and not dummy
            store_right_half<M::W, M::N2 - M::W>(state_g, lane >> KB, pe);
    }
}

inline void mid_kernel_configure()
{
    static_assert(MidDev<1>::Smem <= 232448 && MidDev<2>::Smem <= 232448, "k_mid's shared memory must fit one SM");
    for (SampleKind k : kSampleKinds)
        with_sample_type(k, [](auto t) {
            using T = typename decltype(t)::type;
            cudaFuncSetAttribute(k_mid<T, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MidDev<1>::Smem);
            cudaFuncSetAttribute(k_mid<T, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MidDev<2>::Smem);
        });
}

// kb: 1 -> n = 1024 (groups of two runs), 2 -> n = 512 (groups of four)
inline int mid_launch(cudaStream_t stream, const LongRun *d_runs, uint32_t n_groups, const float *d_pack, int sm_count, SampleKind kind, int kb)
{
    if (!n_groups) return 0;
    const uint32_t grid = static_deal_grid(n_groups, kLongWarps, sm_count);
    if (kb == 1) {
        switch (kind) {
        case kSampleI16: k_mid<int16_t, 1><<<grid, kLongWarps * 32, MidDev<1>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleF16: k_mid<__half, 1><<<grid, kLongWarps * 32, MidDev<1>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleI32: k_mid<int32_t, 1><<<grid, kLongWarps * 32, MidDev<1>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleI24: k_mid<i24, 1><<<grid, kLongWarps * 32, MidDev<1>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        default: k_mid<float, 1><<<grid, kLongWarps * 32, MidDev<1>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        }
    } else {
        switch (kind) {
        case kSampleI16: k_mid<int16_t, 2><<<grid, kLongWarps * 32, MidDev<2>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleF16: k_mid<__half, 2><<<grid, kLongWarps * 32, MidDev<2>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleI32: k_mid<int32_t, 2><<<grid, kLongWarps * 32, MidDev<2>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        case kSampleI24: k_mid<i24, 2><<<grid, kLongWarps * 32, MidDev<2>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        default: k_mid<float, 2><<<grid, kLongWarps * 32, MidDev<2>::Smem, stream>>>(d_runs, n_groups, d_pack); break;
        }
    }
    return cudaGetLastError() != cudaSuccess;
}
#endif  // __CUDACC__

}  // namespace lwb
