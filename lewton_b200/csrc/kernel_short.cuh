// kernel_short.cuh -- fused IMDCT + window + overlap-add for runs of consecutive SHORT blocks of
// n = 256 (blocksize_0 = 8, the short block of every 44.1 / 48 kHz Vorbis stream): the register-resident
// counterpart of kernel_long.cuh for the 6-bit index space.
//
// A 256-point block has 64 complex values z_c = U[2c+1] + i U[2c]; a warp holds 512, so it transforms
// EIGHT consecutive packets of one channel (an "octet") in lockstep: lane = 4 b + l, block b = lane >> 2,
// and the 4 lanes of a block hold its 64 values as 2 groups x 8 slots, exactly the per-lane shape of the
// long kernel.  The step-3 stages are a radix-2 DIF FFT over the 6 bits of c: step 2 flips bit 5, stages
// 0 and 1 flip bits 4 and 3, ld654 covers bits 2, 1, 0 (imdct.rs:385-484), so there are only two phases:
//     phase A: slot = bits 5,4,3  -> step 0, step 2, stages 0, 1              (imdct.rs:337-452)
//     phase C: slot = bits 2,1,0  -> ld654, bit-reverse (renaming), step 7, step 8, window / OLA
// with ONE shared-memory transpose in between (conflict-free for the eight blocks together).  Everything
// else follows the long kernel: the reference's rounding DAG operation for operation, written on
// (group a, group b) pairs of uncontracted IEEE RN operations, twiddles from a per-lane pack, spectrum
// tiles by 1-D TMA into a per-warp ring.
// Eight consecutive packets are 1024 consecutive PCM samples: block b's previous right half (the only
// inter-packet state, audio.rs:847-861) is block b-1's p_even, fetched from the neighbouring lanes by
// shuffle; block 0 takes it from the previous octet (registers) or the stream state (first octet).
//
// The lane functions compile for the host too: tests/emu/short_emu.cpp runs the 32 lanes sequentially
// against the oracle (index maps, swizzle, twiddle pack, bank conflicts) without a GPU.
#pragma once
#include "kernel_long.cuh"

namespace lwb {

constexpr int kShortBs = 8;
constexpr int kShortN = 256;
constexpr int kShortN2 = 128;
constexpr int kShortOct = 8;               // blocks a warp transforms together

struct alignas(16) ShortRun {              // 48 bytes
    const float *in;        // first packet's spectrum (128 floats); next packet at +in_stride
    void *out;              // first emitted packet's PCM (elements of the batch's format); next at +128
    float *state;           // stream state row of this channel (>= 128 floats)
    uint32_t in_stride;
    uint32_t n_packets;     // including a primer packet (has_prev == 0: packet 0 emits nothing)
    uint8_t has_prev;       // 1: packet 0 overlaps with state[0..128)
    uint8_t write_state;    // 1: store the last packet's right half to end_ptr[0..128) (`state` if end_ptr is null)
    uint8_t tail;           // 1: a long block follows whose kernel ran BEFORE this one (LongRun::first_short == 2): end_ptr
                            //    holds its windowed left slope x[ls + i] w[i]; this run adds its right half's share and
                            //    stores the 128 samples the two blocks overlap in, right behind its own PCM (audio.rs:1112-1118)
    uint8_t pad[5];
    float *end_ptr;
};
static_assert(sizeof(ShortRun) == 48, "ShortRun layout");

// the short pack = kernel_long's pack layout without its phase-B slots
constexpr int kSpShift = P_B_END - P_A_END;
LWB_HD constexpr int sp_of(int slot) { return slot < P_A_END ? slot : slot - kSpShift; }
constexpr int SP_END = P_END - kSpShift;                       // 71
constexpr int kShortPackFloats = SP_END * 32 * 2;

// Which complex element of its block sits in (l, slot, half), l = lane & 3
LWB_HD int elemA_s(int l, int slot, int half) { return (half ? 7 - l : l) + 8 * slot; }
LWB_HD int elemC_s(int l, int slot, int half)
{
    const int T = half ? 7 - rev3(l) : rev3(l);
    return 8 * T + slot;
}
// output index m (0..63) of (l, slot, half) AFTER the step-7 half swap of even slots
LWB_HD int outIndex_s(int l, int slot, int half)
{
    const int flip = (slot & 1) ? half : !half;
    return 8 * rev3(slot) + (flip ? 7 - l : l);
}
// word index of complex element c of block b inside a 512-word transpose plane: bank = 4 b + (c1c0 ^ c5c4),
// distinct over the 32 lanes both when they vary (b, c1c0) -- phase A stores -- and (b, c5c4) -- phase C loads
LWB_HD int swzS(int b, int c) { return ((c >> 2) << 5) | (b << 2) | ((c & 3) ^ ((c >> 4) & 3)); }

// Host: per-lane pack from the blocksize-8 tables (a, b: 128; c: 64; w: 128).  Only l = lane & 3 matters.
inline void short_build_pack(const float *a, const float *b, const float *c, const float *w, float *pack)
{
    V *P = reinterpret_cast<V *>(pack);
    for (int lane = 0; lane < 32; lane++) {
        const int l = lane & 3;
        auto put = [&](int slot, float x, float y) { P[sp_of(slot) * 32 + lane] = V{x, y}; };
        float tx[2], ty[2];
        for (int j = 0; j < 8; j++) {                          // step 0 (imdct.rs:337-371)
            for (int h = 0; h < 2; h++) {
                const int cc = elemA_s(l, j, h);
                const float s = cc < 32 ? -1.0f : 1.0f;        // (-x)*A == x*(-A)
                tx[h] = s * a[126 - 2 * cc];
                ty[h] = s * a[127 - 2 * cc];
            }
            put(P_S0W0 + j, tx[0], tx[1]);
            put(P_S0W1 + j, ty[0], ty[1]);
        }
        for (int j = 0; j < 4; j++) {                          // step 2 (imdct.rs:385-430)
            for (int h = 0; h < 2; h++) {
                const int cc = elemA_s(l, j, h);
                tx[h] = a[124 - 4 * cc];
                ty[h] = a[125 - 4 * cc];
            }
            put(P_S2W0 + j, tx[0], tx[1]);
            put(P_S2W1 + j, ty[0], ty[1]);
        }
        for (int u = 0; u < 2; u++) {                          // stage 0: a = r * 8, r < n >> 4
            for (int h = 0; h < 2; h++) {
                const int r = (~elemA_s(l, 2 + u, h)) & 15;
                tx[h] = a[8 * r];
                ty[h] = a[8 * r + 1];
            }
            put(P_L0W0 + u, tx[0], tx[1]);
            put(P_L0W1 + u, ty[0], ty[1]);
        }
        for (int h = 0; h < 2; h++) {                          // stage 1: a = r * 16, r < n >> 5
            const int r = (~elemA_s(l, 1, h)) & 7;
            tx[h] = a[16 * r];
            ty[h] = a[16 * r + 1];
        }
        put(P_L1W0, tx[0], tx[1]);
        put(P_L1W1, ty[0], ty[1]);
        put(P_A2, a[kShortN >> 3], a[kShortN >> 3]);
        for (int jj = 0; jj < 4; jj++) {                       // step 7 (imdct.rs:533-580)
            for (int h = 0; h < 2; h++) {
                const int p = 63 - rev6(elemC_s(l, 2 * jj + 1, h));
                tx[h] = c[2 * p];
                ty[h] = c[2 * p + 1];
            }
            put(P_S7C0 + jj, tx[0], tx[1]);
            put(P_S7C1 + jj, ty[0], ty[1]);
        }
        for (int j = 0; j < 8; j++) {                          // step 8 + window
            float b0[2], b1[2], wl[2], wh[2];
            for (int h = 0; h < 2; h++) {
                const int m = outIndex_s(l, j, h);
                const int cp = 63 - m;
                b0[h] = b[2 * cp];
                b1[h] = b[2 * cp + 1];
                wl[h] = w[m];
                wh[h] = w[127 - m];
            }
            put(P_B0 + j, b0[0], b0[1]);
            put(P_B1 + j, b1[0], b1[1]);
            put(P_WLO + j, wl[0], wl[1]);
            put(P_WHI + j, wh[0], wh[1]);
        }
    }
}

// Phase A for one block.  tile = the block's 128 spectrum floats.  Quad #f yields element c = f from
// (q1, q3) and c = 63 - f from (q0, q2); the lane reads quads #(l + 8 m) and #(7 - l + 8 m), m < 4: they
// feed slots m and 7 - m of both groups.  Then step 2 (bit 5), stage 0 (bit 4), stage 1 (bit 3).
template <class TW>
LWB_HD void phase_a_s(const float *tile, int l, TW tw, V O[8], V E[8])
{
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const Q4 f1 = ld_q4(tile + 4 * (l + 8 * m));
        const Q4 f2 = ld_q4(tile + 4 * (7 - l + 8 * m));
        {
            const V w0 = tw(P_S0W0 + m), w1 = tw(P_S0W1 + m);
            const V qa = V{f1.w, f2.w}, qb = V{f1.y, f2.y};
            O[m] = vsub_p(vmul(qa, w0), vmul(qb, w1));
            E[m] = vadd_p(vmul(qa, w1), vmul(qb, w0));
        }
        {
            const int j = 7 - m;
            const V w0 = tw(P_S0W0 + j), w1 = tw(P_S0W1 + j);
            const V qa = V{f2.x, f1.x}, qb = V{f2.z, f1.z};
            O[j] = vsub_p(vmul(qa, w0), vmul(qb, w1));
            E[j] = vadd_p(vmul(qa, w1), vmul(qb, w0));
        }
    }
#pragma unroll
    for (int j = 0; j < 4; j++) bfly(O[j + 4], E[j + 4], O[j], E[j], tw(P_S2W0 + j), tw(P_S2W1 + j));
#pragma unroll
    for (int u = 0; u < 2; u++) {
        const V w0 = tw(P_L0W0 + u), w1 = tw(P_L0W1 + u);
        bfly(O[2 + u], E[2 + u], O[u], E[u], w0, w1);
        bfly(O[6 + u], E[6 + u], O[4 + u], E[4 + u], w0, w1);
    }
    {
        const V w0 = tw(P_L1W0), w1 = tw(P_L1W1);
#pragma unroll
        for (int j = 1; j < 8; j += 2) bfly(O[j], E[j], O[j - 1], E[j - 1], w0, w1);
    }
}

// step 8 for one slot (imdct.rs:589-658):  p_odd = x[m] = -x[127-m],  p_even = x[128+m] = x[255-m]
LWB_HD void step8_s(V b0, V b1, V Oj, V Ej, V &p_odd, V &p_even)
{
    p_odd = vsub_p(vmul(Oj, b1), vmul(Ej, b0));
    p_even = vnsub_p(vmul(Oj, b0), vmul(Ej, b1));
}
// window / overlap-add (audio.rs:1112-1118):  pcm[m] = x[m] w[m] + prev[m] w[127-m],
// pcm[127-m] = (-p_odd) w[127-m] + prev[127-m] w[m]
LWB_HD void ola_s(V p_odd, V wlo, V whi, V prev_lo, V prev_hi, V &pcm_lo, V &pcm_hi)
{
    pcm_lo = vadd_p(vmul(p_odd, wlo), vmul(prev_lo, whi));
    pcm_hi = vsub_p(vmul(prev_hi, wlo), vmul(p_odd, whi));
}

#if defined(__CUDACC__)
#ifndef LWB_SHORT_WARPS
#define LWB_SHORT_WARPS 8
#endif
#ifndef LWB_SHORT_RING
#define LWB_SHORT_RING 3
#endif
// short-pack slots [kSTwReg0, kSTwReg1) live in registers for the whole kernel
#ifndef LWB_STW_REG0
#define LWB_STW_REG0 0
#endif
#ifndef LWB_STW_REG1
#define LWB_STW_REG1 30
#endif
constexpr int kShortWarps = LWB_SHORT_WARPS;
constexpr int kShortRing = LWB_SHORT_RING;
constexpr int kSTwReg0 = LWB_STW_REG0, kSTwReg1 = LWB_STW_REG1;
constexpr int kShortTileStride = 576;                         // bytes between the blocks' tiles of a stage when they are copied
                                                              // one by one: 512 + 64, so that the LDS.128 of a quarter warp
                                                              // (2 blocks x 4 lanes) hit 8 bank groups; contiguous input
                                                              // (one channel) arrives in one copy at stride 512
constexpr int kShortStateOff = kShortOct * kShortTileStride;  // 4608: the run's state row (first octet of a run with history)
constexpr int kShortStageBytes = 5120;                        // 4608 + 512; the first 4096 bytes double as the transpose scratch
                                                              // and then as the PCM staging; a multiple of 1024 (XOR addressing)
constexpr int kShortFetch = 3;                                // run descriptors are fetched this many runs ahead of the producer
constexpr int kShortDescSlots = kShortFetch + kShortRing + 2; // descriptor slots a fetch may be ahead of the consumer
constexpr size_t kShortSmemBytes = 1024 + (size_t)kShortWarps * kShortRing * kShortStageBytes + (size_t)kShortPackFloats * 4 +
                                   (size_t)kShortWarps * kShortDescSlots * sizeof(ShortRun) + kShortWarps * kShortRing * 8 + 64;

struct TwShort {
    const V *r;                   // registers: short-pack slots [kSTwReg0, kSTwReg1)
    const V *lane_base;           // &pack[lane] in shared memory
    __device__ __forceinline__ V operator()(int slot) const
    {
        const int s = sp_of(slot);
        return (s >= kSTwReg0 && s < kSTwReg1) ? r[s - kSTwReg0] : lane_base[s * 4];
    }
};

// The CTA's shared window of k_short and k_short_g, 1 KB aligned: [ring: warps x Ring stages of StageBytes][pack]
// [descriptors: DescBytes per warp][mbarriers: Ring per warp]
template <int Ring, size_t StageBytes, size_t DescBytes>
struct ShortSmem {
    static constexpr size_t kRingBytes = (size_t)kShortWarps * Ring * StageBytes;
    unsigned char *ring, *s_desc;
    V *s_pack;
    uint64_t *bars;
    __device__ __forceinline__ ShortSmem(unsigned char *smem_raw, int warp)
    {
        unsigned char *base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
        unsigned char *tail = base + kRingBytes + (size_t)kShortPackFloats * 4;
        ring = base + (size_t)warp * Ring * StageBytes;
        s_pack = reinterpret_cast<V *>(base + kRingBytes);
        s_desc = tail + (size_t)warp * DescBytes;
        bars = reinterpret_cast<uint64_t *>(tail + (size_t)kShortWarps * DescBytes) + warp * Ring;
    }
};

// The CTA set-up of k_short and k_short_g: stage the pack, init the first n_bars mbarriers of every warp, and load the
// lane's resident twiddles (short-pack slots [kSTwReg0, kSTwReg1)) into twR.  The pack depends on l = lane & 3 only: the
// shared copy keeps 4 lanes per slot (32 bytes), so that a warp's twiddle read is one multicast wavefront instead of two.
__device__ __forceinline__ void short_cta_setup(const float *pack, V *s_pack, uint64_t *bars, int n_bars, int lane, V *twR)
{
    for (int i = threadIdx.x; i < SP_END * 4; i += blockDim.x)
        s_pack[i] = reinterpret_cast<const V *>(pack)[(i >> 2) * 32 + (i & 3)];
    if (lane == 0) {
        for (int i = 0; i < n_bars; i++) mbar_init(smem_u32(&bars[i]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
#pragma unroll
    for (int s = kSTwReg0; s < kSTwReg1; s++) twR[s - kSTwReg0] = s_pack[s * 4 + (lane & 3)];
}
constexpr int kSTwRegs = kSTwReg1 - kSTwReg0 > 0 ? kSTwReg1 - kSTwReg0 : 1;

// PCM staging: one sample as OutT (samples.rs:86-103).  An i24 sample is staged as its 4-byte integer (stage_esz) and
// packed on the way out.
template <typename OutT>
constexpr uint32_t stage_esz = std::is_same_v<OutT, i24> ? 4u : (uint32_t)sizeof(OutT);
__device__ __forceinline__ void sts_pcm(uint32_t addr, float v, float *) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
// integer and 2-byte samples differ only in the conversion: one staging store per staged size
template <typename OutT>
__device__ __forceinline__ void sts_pcm(uint32_t addr, float v, OutT *)
{
    const auto s = d_sample(v, static_cast<OutT *>(nullptr));
    if constexpr (sizeof(s) == 4) {
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"((uint32_t)s) : "memory");
    } else {
        static_assert(sizeof(s) == 2, "2-byte samples");
        asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(*reinterpret_cast<const unsigned short *>(&s)) : "memory");
    }
}
// four staged samples of one lane -> global, streaming: one 16-byte (f32, i32) or 8-byte (2-byte samples) store; i24:
// the four integers' low 3 bytes packed into three words, three 4-byte stores (12 bytes per lane: 4-byte aligned only)
template <typename OutT>
__device__ __forceinline__ void copy_out4(OutT *dst, uint32_t src)
{
    if constexpr (std::is_same_v<OutT, i24>) {
        uint32_t a, b, c, d;
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(src) : "memory");
        unsigned int *w = reinterpret_cast<unsigned int *>(dst);
        __stcs(w, __byte_perm(a, b, 0x4210));          // a0 a1 a2 b0
        __stcs(w + 1, __byte_perm(b, c, 0x5421));      // b1 b2 c0 c1
        __stcs(w + 2, __byte_perm(c, d, 0x6542));      // c2 d0 d1 d2
    } else if constexpr (sizeof(OutT) == 4) {
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(src) : "memory");
        __stcs(reinterpret_cast<float4 *>(dst), v);
    } else {
        static_assert(sizeof(OutT) == 2, "2-byte samples");
        uint2 v;
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(src) : "memory");
        __stcs(reinterpret_cast<uint2 *>(dst), v);
    }
}

// Transpose addresses (bytes inside the stage; E plane at +0, O plane at +2048).  4 * swzS(b, c) splits into a lane part,
// an additive slot part (an immediate of the access) and a slot part XORed into bits 2..3 -- the stage bases are
// 1024-byte aligned, so that XOR can be applied to the full address:
//   phase A, c = cl + 8 j:   lane part 4 * swzS(b, cl),   + (j << 8),         ^ 4 * (j >> 1)
//   phase C, c = 8 T + j:    lane part 4 * swzS(b, 8 T),  + ((j >> 2) << 7),  ^ 4 * (j & 3)
// PCM staging: sample m of block b sits in row b (128 samples) at chunk (m >> 2) ^ b, position m & 3 -- the XOR with b
// spreads the eight blocks' equal sample indices over the banks.  Lane parts for positions l and 3 - l; the chunk of a
// slot is a compile-time constant XORed in.
template <typename OutT>
struct ShortLanes {
    uint32_t wA0, wA1, wC0, wC1, wP0, wP1;
    __device__ __forceinline__ ShortLanes(int l, int blk)
    {
        constexpr uint32_t ESZ = stage_esz<OutT>;
        wA0 = 4u * (uint32_t)swzS(blk, elemA_s(l, 0, 0)); wA1 = 4u * (uint32_t)swzS(blk, elemA_s(l, 0, 1));
        wC0 = 4u * (uint32_t)swzS(blk, elemC_s(l, 0, 0)); wC1 = 4u * (uint32_t)swzS(blk, elemC_s(l, 0, 1));
        wP0 = (128u * ESZ + 4u * ESZ) * (uint32_t)blk + ESZ * (uint32_t)l;
        wP1 = (128u * ESZ + 4u * ESZ) * (uint32_t)blk + ESZ * (uint32_t)(3 - l);
    }
};

// the one transpose, phase A -> phase C (k_short, k_short_g); the stage is the scratch
template <typename OutT>
__device__ __forceinline__ void transpose_s(const ShortLanes<OutT> &ln, uint32_t stage_s, V O[8], V E[8])
{
    __syncwarp();           // every lane has consumed its quads: the stage becomes the scratch
    {
        const uint32_t a0 = stage_s + ln.wA0, a1 = stage_s + ln.wA1;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            sts_eo(((a0 ^ (4u * (j >> 1))) + (j << 8)), E[j].x, O[j].x);
            sts_eo(((a1 ^ (4u * (j >> 1))) + (j << 8)), E[j].y, O[j].y);
        }
    }
    __syncwarp();
    {
        const uint32_t c0 = stage_s + ln.wC0, c1 = stage_s + ln.wC1;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            lds_eo(((c0 ^ (4u * (j & 3))) + ((j >> 2) << 7)), E[j].x, O[j].x);
            lds_eo(((c1 ^ (4u * (j & 3))) + ((j >> 2) << 7)), E[j].y, O[j].y);
        }
    }
    __syncwarp();           // scratch consumed: the same bytes now take the PCM staging
}

// stage slot j's four samples: odd slots hold sample 8 r + l in .x and 8 r + 7 - l in .y, even slots the other way round
template <typename OutT>
__device__ __forceinline__ void stage_pcm_slot(const ShortLanes<OutT> &ln, uint32_t stage_s, int j, V lo, V hi)
{
    constexpr uint32_t CH = 4u * stage_esz<OutT>;
    const uint32_t p0 = stage_s + ln.wP0, p1 = stage_s + ln.wP1;
    const int r = rev3(j);
    const uint32_t cA = CH * (2 * r), cB = CH * (2 * r + 1), cC = CH * (31 - 2 * r), cD = CH * (30 - 2 * r);
    if (j & 1) {
        sts_pcm(p0 ^ cA, lo.x, (OutT *)nullptr); sts_pcm(p1 ^ cB, lo.y, (OutT *)nullptr);
        sts_pcm(p1 ^ cC, hi.x, (OutT *)nullptr); sts_pcm(p0 ^ cD, hi.y, (OutT *)nullptr);
    } else {
        sts_pcm(p1 ^ cB, lo.x, (OutT *)nullptr); sts_pcm(p0 ^ cA, lo.y, (OutT *)nullptr);
        sts_pcm(p0 ^ cD, hi.x, (OutT *)nullptr); sts_pcm(p1 ^ cC, hi.y, (OutT *)nullptr);
    }
}

// a run's end state: the lane's share of the last block's right half, x[128+m] == x[255-m] (imdct.rs:622-649)
__device__ __forceinline__ void store_end_state_s(float *end_ptr, int l, const V pe[8])
{
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int mx = outIndex_s(l, j, 0), my = outIndex_s(l, j, 1);
        end_ptr[mx] = pe[j].x; end_ptr[my] = pe[j].y;
        end_ptr[127 - mx] = pe[j].x; end_ptr[127 - my] = pe[j].y;
    }
}

// The end of a run whose last block a long block follows, the long block's kernel having run BEFORE this one
// (ShortRun::tail): pcm[i] = x_long[ls + i] w[i] + prev[i] w[127 - i].  The first product comes from the long kernel at
// end_ptr, prev is this block's right half (prev[m] == prev[127 - m] == p_even); the 128 samples go to `on`.
template <typename OutT>
__device__ __forceinline__ void short_tail(const TwShort &tw, int l, const V pe[8], const float *end_ptr, OutT *on)
{
    float cw[8][4];                              // all loads first: the stores below may alias them as far as the compiler knows
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int mx = outIndex_s(l, j, 0), my = outIndex_s(l, j, 1);
        cw[j][0] = __ldcg(end_ptr + mx); cw[j][1] = __ldcg(end_ptr + my);
        cw[j][2] = __ldcg(end_ptr + 127 - mx); cw[j][3] = __ldcg(end_ptr + 127 - my);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int mx = outIndex_s(l, j, 0), my = outIndex_s(l, j, 1);
        const V wlo = tw(P_WLO + j), whi = tw(P_WHI + j);
        st_pcm(on + mx, __fadd_rn(cw[j][0], __fmul_rn(pe[j].x, whi.x)));
        st_pcm(on + my, __fadd_rn(cw[j][1], __fmul_rn(pe[j].y, whi.y)));
        st_pcm(on + 127 - mx, __fadd_rn(cw[j][2], __fmul_rn(pe[j].x, wlo.x)));
        st_pcm(on + 127 - my, __fadd_rn(cw[j][3], __fmul_rn(pe[j].y, wlo.y)));
    }
}

// runs: one descriptor per run; pack: short_build_pack of the setup's blocksize-8 tables.
//
// Short-block runs are short -- a burst between long blocks is one octet --, so the per-run latencies must overlap with
// the previous runs' arithmetic: kernel_deal.cuh's static-deal driver, one run per item, one octet per unit (TMA copies
// of up to eight 512-byte spectrum blocks -- one copy when the blocks are contiguous --, plus the 512-byte state row in
// front of a run with history, all counted on the stage's mbarrier).
// PCM leaves through shared memory: the lanes' samples are staged (swizzled, conflict-free) and go out as one
// 128-bit (f32) / 64-bit (i16) store per lane and packet, 512 / 256 contiguous bytes per instruction, instead of
// 16-byte pieces of eight different lines per instruction, which made the L1 data pipe the limiter.
template <typename OutT>
__global__ void __launch_bounds__(kShortWarps * 32, 1)
k_short(const ShortRun *__restrict__ runs, uint32_t n_runs, const float *__restrict__ pack)
{
    extern __shared__ __align__(128) unsigned char smem_s[];
    constexpr uint32_t ESZ = stage_esz<OutT>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int l = lane & 3, blk = lane >> 2;
    const ShortSmem<kShortRing, kShortStageBytes, kShortDescSlots * sizeof(ShortRun)> sm(smem_s, warp);
    unsigned char *ring = sm.ring;
    uint4 *s_desc = reinterpret_cast<uint4 *>(sm.s_desc);
    V twR[kSTwRegs];
    short_cta_setup(pack, sm.s_pack, sm.bars, kShortRing, lane, twR);
    const TwShort tw{twR, sm.s_pack + l};
    const ShortLanes<OutT> ln(l, blk);

    const uint32_t W = gridDim.x * kShortWarps, gw = blockIdx.x * kShortWarps + warp;
    if (gw >= n_runs) return;
    StaticDeal<3, kShortDescSlots, kShortFetch, kShortRing, kShortStageBytes> deal(
        runs, n_runs, W, gw, smem_u32(s_desc), smem_u32(ring), smem_u32(sm.bars), lane);
    // ShortRun fields inside the three quads: q0 = {in, out}, q1 = {state, in_stride, n_packets}, q2 = {has_prev | write_state << 8, ...}
    auto units = [&](uint32_t sl) { return (s_desc[3 * sl + 1].w + kShortOct - 1) / kShortOct; };
    auto issue = [&](uint32_t sl, uint32_t oct, uint32_t bar, uint32_t dst) {
        const uint4 d0 = s_desc[3 * sl], d1 = s_desc[3 * sl + 1], d2 = s_desc[3 * sl + 2];
        const float *in = reinterpret_cast<const float *>(((unsigned long long)d0.y << 32) | d0.x);
        const float *state = reinterpret_cast<const float *>(((unsigned long long)d1.y << 32) | d1.x);
        const uint32_t in_stride = d1.z, npk = d1.w;
        const bool with_state = oct == 0 && (d2.x & 0xffu);
        const uint32_t nb = min((uint32_t)kShortOct, npk - oct * kShortOct);
        const bool contig = in_stride == (uint32_t)kShortN2;
        if (lane == 0) mbar_expect_tx(bar, (nb + (with_state ? 1u : 0u)) * (uint32_t)(kShortN2 * 4));
        __syncwarp();
        if (contig) {
            if (lane == 0) {
                fence_proxy_async();        // the stage was written through the generic proxy (transpose, staging) before
                tma_load_1d(dst, in + (size_t)(oct * kShortOct) * kShortN2, nb * (uint32_t)(kShortN2 * 4), bar);
            }
        } else if ((uint32_t)lane < nb) {
            fence_proxy_async();
            tma_load_1d(dst + lane * kShortTileStride, in + (size_t)(oct * kShortOct + lane) * in_stride, kShortN2 * 4, bar);
        }
        if (lane == 8 && with_state) {
            fence_proxy_async();
            tma_load_1d(dst + kShortStateOff, state, kShortN2 * 4, bar);
        }
    };
    deal.start(units, issue);

    for (uint32_t c_run = gw; c_run < n_runs; c_run += W) {
        const uint32_t sl = deal.take_slot();
        const uint4 d0 = s_desc[3 * sl], d1 = s_desc[3 * sl + 1], d2 = s_desc[3 * sl + 2];
        OutT *out = reinterpret_cast<OutT *>(((unsigned long long)d0.w << 32) | d0.z);
        float *state = reinterpret_cast<float *>(((unsigned long long)d1.y << 32) | d1.x);
        const uint32_t npk = d1.w;
        const bool has_prev = (d2.x & 0xffu) != 0, write_state = ((d2.x >> 8) & 0xffu) != 0, tail = ((d2.x >> 16) & 0xffu) != 0;
        float *end_ptr = reinterpret_cast<float *>(((unsigned long long)d2.w << 32) | d2.z);
        if (!end_ptr) end_ptr = state;
        const bool contig = d1.z == (uint32_t)kShortN2;
        const uint32_t n_oct = (npk + kShortOct - 1) / kShortOct;
        const uint32_t koff = has_prev ? 0u : 1u;                // packet 0 emits nothing then: packet k lands at 128 (k - 1)

        V carry[8];                                              // p_even of the previous octet (lanes of block 7 matter)
#pragma unroll
        for (int j = 0; j < 8; j++) carry[j] = V{0.f, 0.f};
        V pe[8];
        for (uint32_t o = 0; o < n_oct; o++) {
            const uint32_t stage = deal.wait_stage();
            const uint32_t stage_s = deal.ring_s + stage * kShortStageBytes;
            const unsigned char *stage_p = ring + stage * kShortStageBytes;
            V O[8], E[8];
            phase_a_s(reinterpret_cast<const float *>(stage_p + blk * (contig ? kShortN2 * 4 : kShortTileStride)), l, tw, O, E);
            const bool first0 = (o == 0 && blk == 0);
            transpose_s(ln, stage_s, O, E);
            phase_c_fft<1>(tw, &O, &E);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                V p_odd;
                step8_s(tw(P_B0 + j), tw(P_B1 + j), O[j], E[j], p_odd, pe[j]);
                // previous block's right half: block b-1 of this octet sits 4 lanes down; block 0 takes the last block of
                // the previous octet, which the lanes of block 7 (whose own p_even nobody needs before the next octet)
                // put on the same shuffle
                const V src = blk == 7 ? carry[j] : pe[j];
                V plo;
                plo.x = __shfl_sync(0xffffffffu, src.x, (lane + 28) & 31);
                plo.y = __shfl_sync(0xffffffffu, src.y, (lane + 28) & 31);
                V phi = plo;
                if (first0 && has_prev) {                        // the stream state (an imported one need not be symmetric);
                    const int mx = outIndex_s(l, j, 0), my = outIndex_s(l, j, 1);      // its tile lies beyond the scratch / staging bytes
                    const uint32_t sa = stage_s + kShortStateOff;
                    plo = V{lds_f32(sa + 4 * mx), lds_f32(sa + 4 * my)};
                    phi = V{lds_f32(sa + 4 * (127 - mx)), lds_f32(sa + 4 * (127 - my))};
                }
                V lo, hi;
                ola_s(p_odd, tw(P_WLO + j), tw(P_WHI + j), plo, phi, lo, hi);
                stage_pcm_slot(ln, stage_s, j, lo, hi);
            }
#pragma unroll
            for (int j = 0; j < 8; j++) carry[j] = pe[j];
            __syncwarp();
            // one packet per instruction: lane L copies samples [4 L, 4 L + 4) of packet 8 o + i
            {
                const uint32_t nb = min((uint32_t)kShortOct, npk - o * kShortOct);
                OutT *og = out + (ptrdiff_t)((int)(o * kShortOct) - (int)koff) * kShortN2 + 4 * lane;
#pragma unroll
                for (int i = 0; i < kShortOct; i++) {
                    if ((uint32_t)i < nb && !(o == 0 && i == 0 && !has_prev))
                        copy_out4(og + i * kShortN2, stage_s + (128u * ESZ) * i + (4u * ESZ) * (uint32_t)(lane ^ i));
                }
            }
            __syncwarp();                                        // staging and state tile consumed: the stage is free
            deal.produce(units, issue);
            deal.next_stage();
        }
        const bool last = (uint32_t)blk == ((npk - 1) & (kShortOct - 1));
        if (write_state && last) store_end_state_s(end_ptr, l, pe);
        if (tail && last) short_tail(tw, l, pe, end_ptr, out + (size_t)(npk - koff) * kShortN2);
    }
}

// ---------------------------------------------------------------------------------------------
// k_short_g: bursts.  Between two long blocks a stream has one to a few short blocks; k_short would spend a whole octet
// iteration on each such run with one or two of its eight block positions occupied.  Here the eight block positions of
// a warp belong to EIGHT DIFFERENT runs of equal length (a "group"; the host sorts the short runs by length and pads
// each length class with dummies) which advance in lockstep, one packet per iteration -- so block position b's previous
// right half is simply its own p_even of the iteration before (registers, no shuffle), or its run's state tile in
// iteration 0.  Descriptors: 8 ShortRun per group (dummy: in == nullptr).  The static-deal driver of k_short with one
// group per item and one packet per unit; a stage carries the eight state tiles behind the eight spectrum tiles.
// ---------------------------------------------------------------------------------------------
constexpr int kShortGRing = 2;
constexpr int kShortGStageBytes = kShortOct * kShortTileStride + kShortOct * kShortN2 * 4 + 512;     // 4608 + 4096 -> 9216 (1024-aligned)
constexpr int kShortGFetch = 2;
constexpr int kShortGDescSlots = kShortGFetch + kShortGRing + 3;
constexpr size_t kShortGDescBytes = (size_t)kShortOct * sizeof(ShortRun);                                  // 384
constexpr size_t kShortGSmemBytes = 1024 + (size_t)kShortWarps * kShortGRing * kShortGStageBytes + (size_t)kShortPackFloats * 4 +
                                    (size_t)kShortWarps * kShortGDescSlots * kShortGDescBytes + kShortWarps * kShortGRing * 8 + 64;
static_assert(kShortGStageBytes % 1024 == 0, "XOR addressing of the transposes needs 1024-aligned stages");

template <typename OutT>
__global__ void __launch_bounds__(kShortWarps * 32, 1)
k_short_g(const ShortRun *__restrict__ runs, uint32_t n_groups, const float *__restrict__ pack)
{
    extern __shared__ __align__(128) unsigned char smem_s[];
    constexpr uint32_t ESZ = stage_esz<OutT>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int l = lane & 3, blk = lane >> 2;
    const ShortSmem<kShortGRing, kShortGStageBytes, kShortGDescSlots * kShortGDescBytes> sm(smem_s, warp);
    unsigned char *ring = sm.ring;
    ShortRun *s_desc = reinterpret_cast<ShortRun *>(sm.s_desc);
    V twR[kSTwRegs];
    short_cta_setup(pack, sm.s_pack, sm.bars, kShortGRing, lane, twR);
    const TwShort tw{twR, sm.s_pack + l};
    const ShortLanes<OutT> ln(l, blk);
    constexpr uint32_t kStateOff = kShortOct * kShortTileStride;               // state tile of block b at + 512 b

    const uint32_t W = gridDim.x * kShortWarps, gw = blockIdx.x * kShortWarps + warp;
    if (gw >= n_groups) return;
    StaticDeal<kShortGDescBytes / 16, kShortGDescSlots, kShortGFetch, kShortGRing, kShortGStageBytes> deal(
        runs, n_groups, W, gw, smem_u32(s_desc), smem_u32(ring), smem_u32(sm.bars), lane);
    auto units = [&](uint32_t sl) { return s_desc[sl * kShortOct].n_packets; };
    auto issue = [&](uint32_t sl, uint32_t t, uint32_t bar, uint32_t dst) {     // lane b < 8 issues block position b's copies
        const ShortRun *g = s_desc + sl * kShortOct;
        const bool mine = lane < kShortOct && g[lane & 7].in != nullptr;
        const bool st = mine && t == 0 && g[lane & 7].has_prev;
        const uint32_t n_tiles = (uint32_t)__popc(__ballot_sync(0xffffffffu, mine)) + (uint32_t)__popc(__ballot_sync(0xffffffffu, st));
        if (lane == 0) mbar_expect_tx(bar, n_tiles * (uint32_t)(kShortN2 * 4));
        __syncwarp();
        if (mine) {
            fence_proxy_async();
            tma_load_1d(dst + lane * kShortTileStride, g[lane].in + (size_t)t * g[lane].in_stride, kShortN2 * 4, bar);
            if (st) tma_load_1d(dst + kStateOff + lane * (kShortN2 * 4), g[lane].state, kShortN2 * 4, bar);
        }
    };
    deal.start(units, issue);

    for (uint32_t c_grp = gw; c_grp < n_groups; c_grp += W) {
        // (the descriptor slot of the group being consumed is never the target of a fetch)
        const ShortRun *g = s_desc + deal.take_slot() * kShortOct;
        const uint32_t npk = g[0].n_packets;
        const bool valid = g[blk].in != nullptr, has_prev = valid && g[blk].has_prev;
        uint32_t emit0 = 0;               // bit i: position i emits in iteration 0; bit 8 + i: position i is not a dummy
#pragma unroll
        for (int i = 0; i < kShortOct; i++)
            if (g[i].in != nullptr) emit0 |= (g[i].has_prev ? 1u : 0u) << i | 256u << i;
        V pe[8];
#pragma unroll
        for (int j = 0; j < 8; j++) pe[j] = V{0.f, 0.f};
        for (uint32_t t = 0; t < npk; t++) {
            const uint32_t stage = deal.wait_stage();
            const uint32_t stage_s = deal.ring_s + stage * kShortGStageBytes;
            const unsigned char *stage_p = ring + stage * kShortGStageBytes;
            V O[8], E[8];
            phase_a_s(reinterpret_cast<const float *>(stage_p + blk * kShortTileStride), l, tw, O, E);
            transpose_s(ln, stage_s, O, E);
            phase_c_fft<1>(tw, &O, &E);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                V p_odd, lo, hi;
                V plo = pe[j];                                   // the position's own right half of the iteration before
                step8_s(tw(P_B0 + j), tw(P_B1 + j), O[j], E[j], p_odd, pe[j]);
                V phi = plo;
                if (t == 0 && has_prev) {                        // the run's state tile (an imported state need not be symmetric);
                    const int mx = outIndex_s(l, j, 0), my = outIndex_s(l, j, 1);      // it lies beyond the scratch / staging bytes
                    const uint32_t sa = stage_s + kStateOff + (uint32_t)blk * (kShortN2 * 4);
                    plo = V{lds_f32(sa + 4 * mx), lds_f32(sa + 4 * my)};
                    phi = V{lds_f32(sa + 4 * (127 - mx)), lds_f32(sa + 4 * (127 - my))};
                }
                ola_s(p_odd, tw(P_WLO + j), tw(P_WHI + j), plo, phi, lo, hi);
                stage_pcm_slot(ln, stage_s, j, lo, hi);
            }
            __syncwarp();
            // one packet per instruction: lane L copies samples [4 L, 4 L + 4) of position i's packet t
#pragma unroll
            for (int i = 0; i < kShortOct; i++) {
                const bool emits = (emit0 >> (8 + i)) & 1u ? (t > 0 || ((emit0 >> i) & 1u)) : false;
                if (emits) {
                    const uint32_t koff = ((emit0 >> i) & 1u) ? 0u : 1u;
                    copy_out4(static_cast<OutT *>(g[i].out) + (size_t)(t - koff) * kShortN2 + 4 * lane,
                              stage_s + (128u * ESZ) * i + (4u * ESZ) * (uint32_t)(lane ^ i));
                }
            }
            __syncwarp();                                        // staging consumed: the stage is free
            deal.produce(units, issue);
            deal.next_stage();
        }
        float *end_ptr = g[blk].end_ptr ? g[blk].end_ptr : g[blk].state;
        if (valid && g[blk].write_state) store_end_state_s(end_ptr, l, pe);
        if (valid && g[blk].tail) short_tail(tw, l, pe, end_ptr, static_cast<OutT *>(g[blk].out) + (size_t)(npk - (has_prev ? 0u : 1u)) * kShortN2);
    }
}

inline int short_launch_groups(cudaStream_t stream, const ShortRun *d_runs, uint32_t n_groups, const float *d_pack, int sm_count, SampleKind kind)
{
    if (!n_groups) return 0;
    const uint32_t grid = static_deal_grid(n_groups, kShortWarps, sm_count);
    switch (kind) {
    case kSampleI16: k_short_g<int16_t><<<grid, kShortWarps * 32, kShortGSmemBytes, stream>>>(d_runs, n_groups, d_pack); break;
    case kSampleF16: k_short_g<__half><<<grid, kShortWarps * 32, kShortGSmemBytes, stream>>>(d_runs, n_groups, d_pack); break;
    case kSampleI32: k_short_g<int32_t><<<grid, kShortWarps * 32, kShortGSmemBytes, stream>>>(d_runs, n_groups, d_pack); break;
    case kSampleI24: k_short_g<i24><<<grid, kShortWarps * 32, kShortGSmemBytes, stream>>>(d_runs, n_groups, d_pack); break;
    default: k_short_g<float><<<grid, kShortWarps * 32, kShortGSmemBytes, stream>>>(d_runs, n_groups, d_pack); break;
    }
    return cudaGetLastError() != cudaSuccess;
}

inline void short_kernel_configure()
{
    for (SampleKind k : kSampleKinds)
        with_sample_type(k, [](auto t) {
            using T = typename decltype(t)::type;
            cudaFuncSetAttribute(k_short<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kShortSmemBytes);
            cudaFuncSetAttribute(k_short_g<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kShortGSmemBytes);
        });
}

inline int short_launch(cudaStream_t stream, const ShortRun *d_runs, uint32_t n_runs, const float *d_pack, int sm_count, SampleKind kind)
{
    if (!n_runs) return 0;
    const uint32_t grid = static_deal_grid(n_runs, kShortWarps, sm_count);
    switch (kind) {
    case kSampleI16: k_short<int16_t><<<grid, kShortWarps * 32, kShortSmemBytes, stream>>>(d_runs, n_runs, d_pack); break;
    case kSampleF16: k_short<__half><<<grid, kShortWarps * 32, kShortSmemBytes, stream>>>(d_runs, n_runs, d_pack); break;
    case kSampleI32: k_short<int32_t><<<grid, kShortWarps * 32, kShortSmemBytes, stream>>>(d_runs, n_runs, d_pack); break;
    case kSampleI24: k_short<i24><<<grid, kShortWarps * 32, kShortSmemBytes, stream>>>(d_runs, n_runs, d_pack); break;
    default: k_short<float><<<grid, kShortWarps * 32, kShortSmemBytes, stream>>>(d_runs, n_runs, d_pack); break;
    }
    return cudaGetLastError() != cudaSuccess;
}
#endif  // __CUDACC__

}  // namespace lwb
