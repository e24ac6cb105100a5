// kernel_prologue.cuh -- the residue entry's front stages for batches (audio.rs:991-1039), as two kernels that
// replace the per-packet-CTA k_prologue of kernels_generic.cuh wherever a batch has <= 8 channels:
//
//   k_floor1_segments : floor-1 step 1 (post unwrap, audio.rs:391-435) with one THREAD per (packet, channel) row --
//                       the unwrap is serial over <= 65 posts, so 32 independent rows per warp is the only way to
//                       keep its lanes busy -- then every flagged segment of the row packed for per-bin evaluation
//                       (floor1_eval.cuh: Seg4, division-free closed form of render_line, audio.rs:503-524);
//   k_prologue_fused  : one CTA per packet, one thread per 4 bins, all channels: the rows' segment tables and a
//                       bin -> segment bitmap in shared memory, floor value per bin (closed form -> dB table,
//                       audio.rs:552-554; unused floor = zero curve, :1021-1024; dense = host-computed floor-0;
//                       zero = floor-0 curve computed by k_floor0_curves),
//                       inverse coupling in registers / shared memory (steps in reverse, audio.rs:991-1002),
//                       multiply (:1035-1037), float4 loads and stores.  The kernel is HBM-bound (4 B in + 4 B out per
//                       coefficient); the per-bin floor arithmetic rides in its idle issue slots.
//
// History: the per-packet-CTA kernel was far from its roofline time (serial unwrap on one lane per warp with the CTA
// waiting, 8-way predicated register arrays).  A first split rendered the curve to a byte arena in a separate kernel
// (16 bins per work item): its per-bin segment-crossing branches diverged and the curve cost 2 B per coefficient of
// extra traffic.
#pragma once
#include "kernels_generic.cuh"

namespace lwb {

constexpr int kSegRows = 64;           // (packet, channel) rows per CTA of k_floor1_segments
constexpr int kSegThreads = 256;
constexpr int kSegStride = LWB_MAX_POSTS + 3;   // 68 Seg4 per row: <= 66 segments (65 posts + flat tail) + sentinel
// per-row bin -> segment index: `words` bitmap words (bit x set <=> a flagged post sits at bin x) followed by `words`
// bytes (flagged posts in the words before); row stride in bytes:
__host__ __device__ inline size_t seg_index_stride(int words) { return ((size_t)words * 5 + 15) & ~(size_t)15; }
inline size_t floor1_segments_smem(int words) { return (size_t)kSegRows * words * sizeof(uint32_t); }

// grid = ceil(n_pk * C / kSegRows).  Row r = (packet ordinal in pkts) * C + channel.
//   seg_cnt[r]  = segments of the row (0 when its floor kind is not LWB_FLOOR_ONE) | 0x80 if any of them needs the
//                 12-bit post-shift (x lists reaching beyond 4096);
//   segtab[r * kSegStride + j], j <= count (the last one a sentinel);   seg_index: see seg_index_stride.
// words = bitmap words per row = (largest n/2 of the batch) / 32.
__global__ void __launch_bounds__(kSegThreads)
k_floor1_segments(const DevPacket *__restrict__ pkts, uint32_t n_rows, int C, const uint8_t *__restrict__ floor_kind,
                  const uint32_t *__restrict__ floor1_y, uint4 *__restrict__ segtab, uint8_t *__restrict__ seg_cnt,
                  unsigned char *__restrict__ seg_index, int words, const uint32_t *__restrict__ magic_tab)
{
    extern __shared__ uint32_t s_bm[];                  // [kSegRows][words]
    __shared__ uint16_t s_x[kSegRows][kSegStride];
    __shared__ uint16_t s_y[kSegRows][kSegStride];
    __shared__ int s_m[kSegRows];
    __shared__ int s_n2[kSegRows];
    __shared__ unsigned int s_flag[kSegRows];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t row0 = blockIdx.x * kSegRows;
    if (tid < kSegRows) {
        const uint32_t row = row0 + tid;
        int m = 0, n2 = 0;
        if (row < n_rows) {
            const uint32_t pk = row / (uint32_t)C, c = row - pk * (uint32_t)C;
            const DevPacket &p = pkts[pk];
            const uint64_t frow = p.pkt_index * (uint64_t)C + c;
            n2 = p.n >> 1;
            if (floor_kind[frow] == LWB_FLOOR_ONE) {
                const DevSetup &su = *p.setup;
                const DevFloor1 &fl = su.floors[su.mappings[p.mapping].floor_of_channel[c]];
                m = d_floor1_posts(fl, floor1_y + frow * LWB_MAX_POSTS, n2, s_x[tid], s_y[tid]);
            }
        }
        s_m[tid] = m;
        s_n2[tid] = n2;
        s_flag[tid] = 0;
    }
    for (int i = tid; i < kSegRows * words; i += kSegThreads) s_bm[i] = 0u;
    __syncthreads();
    for (int i = tid; i < kSegRows * kSegStride; i += kSegThreads) {
        const int r = i / kSegStride, j = i - r * kSegStride;
        const int nseg = s_m[r] - 1;
        if (j <= nseg && nseg > 0) {                    // j == nseg: sentinel = a copy of the last segment
            const int jj = j < nseg ? j : nseg - 1;
            const Seg4 sg = d_floor1_pack_segment(s_x[r], s_y[r], jj, magic_tab);
            segtab[(size_t)(row0 + r) * kSegStride + j] = make_uint4(sg.x, sg.y, sg.z, sg.w);
            if (j < nseg) {
                const int x0 = s_x[r][j];
                if (x0 < s_n2[r]) atomicOr(&s_bm[r * words + (x0 >> 5)], 1u << (x0 & 31));
                if (sg.y & 2u) atomicOr(&s_flag[r], 1u);
            }
        }
    }
    __syncthreads();
    for (int r = warp; r < kSegRows; r += kSegThreads / 32) {
        const uint32_t row = row0 + r;
        if (row >= n_rows) break;
        const int nseg = s_m[r] > 1 ? s_m[r] - 1 : 0;
        if (lane == 0) seg_cnt[row] = (uint8_t)(nseg | (s_flag[r] ? 0x80 : 0));
        if (!nseg) continue;
        unsigned char *ix = seg_index + (size_t)row * seg_index_stride(words);
        uint32_t run = 0;
        for (int w0 = 0; w0 < words; w0 += 32) {
            const uint32_t bits = (w0 + lane < words) ? s_bm[r * words + w0 + lane] : 0u;
            const uint32_t v = (uint32_t)__popc(bits);
            uint32_t inc = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= d) inc += t;
            }
            if (w0 + lane < words) {
                reinterpret_cast<uint32_t *>(ix)[w0 + lane] = bits;
                ix[(size_t)words * 4 + w0 + lane] = (unsigned char)(run + inc - v);
            }
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
}

constexpr int kPfThreads = 256;
constexpr int kPfMaxWords = 128;       // bitmap words per row: n/2 <= 4096 bins
// dynamic shared memory per channel: the row's segment table and bin -> segment index, and (more than one channel)
// the coupling staging
__host__ __device__ inline size_t pf_row_bytes(int words) { return kSegStride * sizeof(uint4) + seg_index_stride(words); }
// vq_elems: channels * (largest n/2) of a LWB_ENTRY_VQ batch (the residue accumulators), else 0
inline size_t prologue_fused_smem(int channels, int words, size_t vq_elems = 0)
{
    // one or two channels, dense residue: two table buffers (the kernel pipelines the packets) -- they fit where the
    // general path keeps its coupling staging
    const size_t staging = channels > 1 ? (size_t)channels * kPfThreads * sizeof(float4) : 0;
    const size_t second = channels <= 2 && !vq_elems ? (size_t)channels * pf_row_bytes(words) : 0;
    return (size_t)channels * pf_row_bytes(words) + (staging > second ? staging : second) + vq_elems * sizeof(float);
}
// device view of a batch's VQ arrays (biased so that absolute packet rows / absolute offsets address them)
struct VqDev { const lwb_vq_run *runs; const uint64_t *run_off; const uint16_t *entries; const uint64_t *ent_off; };
constexpr size_t kVqMaxElems = 12288;          // 48 KB of accumulators: stereo up to n = 8192, 5.1 up to n = 4096

// LWB_ENTRY_VQ: the packet's residue vectors, accumulated in shared memory from its VQ runs in the reference's
// order (residue_packet_decode_inner, audio.rs:620-717; residue_packet_read_partition, :587-618): per coefficient
// the f32 additions happen pass by pass; within a pass the vectors of a packet are disjoint, so the runs of a pass
// go in parallel (one thread per run, its vectors in sequence).  acc: [C][n2], zeroed here.  Called by the whole CTA,
// thread tid of nthreads (k_prologue_fused, k_chain); ends on a CTA barrier.
__device__ __forceinline__ void d_vq_accumulate(float *acc, int C, int n2, const DevSetup &su, const DevMapping &mp,
                                                const lwb_vq_run *__restrict__ runs, uint32_t nruns,
                                                const uint16_t *__restrict__ entries, uint32_t nent, int tid, int nthreads)
{
    const int total = C * n2;
    for (int i = tid; i < total; i += nthreads) acc[i] = 0.f;
    __syncthreads();
    for (uint32_t pass = 0; pass < 8; pass++) {
        for (uint32_t i = tid; i < nruns; i += nthreads) {
            const lwb_vq_run r = runs[i];
            if ((r.pass_kind & 7u) != pass || r.book >= su.n_books) continue;
            const DevBook bk = su.books[r.book];
            const int kind = (r.pass_kind >> 3) & 3, dims = bk.dims;
            if (!bk.vq || !dims || (uint32_t)r.first + r.count > nent) continue;
            const int step = kind == 1 ? (r.aux < su.n_residues ? (int)(su.res_psize[r.aux] / dims) : 0) : 1;
            const int nch = kind == 2 ? (r.aux < LWB_MAX_SUBMAPS ? mp.sub_nch[r.aux] : 0) : 1;
            if (step <= 0 || nch <= 0) continue;
            for (int q = 0; q < r.count; q++) {
                const uint32_t e = entries[r.first + q];
                if (e >= bk.entries) continue;
                const float *__restrict__ v = bk.vq + (size_t)e * dims;
                if (kind == 0) {                               // residue type 1: contiguous (audio.rs:599-615)
                    const int p0 = r.pos + q * dims;
                    if (p0 + dims > total) break;
                    for (int k = 0; k < dims; k++) acc[p0 + k] = __fadd_rn(acc[p0 + k], v[k]);
                } else if (kind == 1) {                        // residue type 0: stride partition_size / dimensions (:589-597)
                    const int p0 = r.pos + q;
                    if (p0 + (dims - 1) * step >= total) break;
                    for (int k = 0; k < dims; k++) acc[p0 + k * step] = __fadd_rn(acc[p0 + k * step], v[k]);
                } else {                                       // residue type 2: one interleaved vector per submap (:744-756)
                    for (int k = 0; k < dims; k++) {
                        const int t = r.pos + q * dims + k, bin = t / nch;
                        if (bin >= n2) break;
                        const int a = mp.sub_ch[r.aux][t - bin * nch] * n2 + bin;
                        acc[a] = __fadd_rn(acc[a], v[k]);
                    }
                }
            }
        }
        __syncthreads();
    }
}

// Floor values of the 4 bins [k0, k0 + 4) of one channel row, tables in shared memory.
template <bool SHIFT>
__device__ __forceinline__ float4 d_floor_quad_one(const float *__restrict__ s_db, const uint4 *__restrict__ tab,
                                                   const unsigned char *__restrict__ ix, int words, int k0)
{
    // segment of bin k = (number of flagged posts with x <= k) - 1.  Post 0 is always flagged (d_floor1_posts), and
    // prepare_floor1 refuses every x list whose post 0 is not at x = 0, so every bin has a segment.  The four bins of a
    // quad share one bitmap word and look their segments up independently of one another.
    const uint32_t bits = reinterpret_cast<const uint32_t *>(ix)[k0 >> 5];
    const int pre = (int)ix[(size_t)words * 4 + (k0 >> 5)] - 1;
    float f[4];
#pragma unroll
    for (int b = 0; b < 4; b++) {
        const uint4 P = tab[pre + __popc(bits & (0xffffffffu >> (31 - ((k0 & 31) + b))))];
        f[b] = s_db[d_floor1_seg_y<SHIFT>(Seg4{P.x, P.y, P.z, P.w}, k0 + b) & 255u];
    }
    return make_float4(f[0], f[1], f[2], f[3]);
}
// zero: the curves k_floor0_curves rendered for LWB_FLOOR_ZERO rows, or nullptr (such rows then act as unused)
__device__ __forceinline__ float4 d_floor_quad(int kind, int cnt, const float *__restrict__ s_db, const uint4 *__restrict__ tab,
                                               const unsigned char *__restrict__ ix, int words, int k0,
                                               const float *__restrict__ dense, const float *__restrict__ zero, uint64_t e)
{
    if (kind == LWB_FLOOR_ONE && (cnt & 0x7f))
        return (cnt & 0x80) ? d_floor_quad_one<true>(s_db, tab, ix, words, k0) : d_floor_quad_one<false>(s_db, tab, ix, words, k0);
    if (kind == LWB_FLOOR_DENSE) return *reinterpret_cast<const float4 *>(dense + e);
    if (kind == LWB_FLOOR_ZERO && zero) return *reinterpret_cast<const float4 *>(zero + e);
    return make_float4(0.f, 0.f, 0.f, 0.f);                       // audio.rs:1021-1024
}

// Header fields of a packet with <= 2 channels and at most one coupling step; kinds, cnt: its rows' floor kinds and
// segment counts
struct PfStereo { int n2, nsteps, k0, k1, c0, c1; bool swapped; uint64_t base; };
__device__ __forceinline__ PfStereo d_pf_stereo_head(const DevPacket &p, const DevMapping &mp, int C, const uint8_t *__restrict__ kinds,
                                                     const uint8_t *__restrict__ cnt)
{
    PfStereo h;
    h.n2 = p.n >> 1;
    h.nsteps = mp.n_coupling;
    h.swapped = h.nsteps == 1 && mp.mag[0] == 1;
    h.base = p.coeff_off;
    h.k0 = kinds[0]; h.k1 = C == 2 ? kinds[1] : LWB_FLOOR_UNUSED;
    h.c0 = cnt[0]; h.c1 = C == 2 ? cnt[1] : 0;
    return h;
}
// Quad q of such a packet: couple the residue quads r0, r1 (audio.rs:991-1002), multiply by the floor values out of
// the rows' tables at `tabs` (row stride rowb), store -- at evict-first priority (STREAM) or plainly.
template <bool STREAM>
__device__ __forceinline__ void d_pf_stereo_quad(const PfStereo &h, int C, int q, float4 r0, float4 r1, const unsigned char *tabs,
                                                 size_t rowb, int words, const float *__restrict__ s_db, const float *__restrict__ dense,
                                                 const float *__restrict__ zero, float *__restrict__ spec)
{
    const uint64_t e0 = h.base + 4 * (uint64_t)q, e1 = e0 + h.n2;
    d_inverse_couple_stereo(h.nsteps, h.swapped, r0, r1);
    const unsigned char *tabs1 = tabs + rowb;
    const float4 f0 = d_floor_quad(h.k0, h.c0, s_db, reinterpret_cast<const uint4 *>(tabs), tabs + kSegStride * 16, words, 4 * q, dense, zero, e0);
    if (STREAM) __stcs(reinterpret_cast<float4 *>(spec + e0), d_floor_mul(f0, r0));
    else *reinterpret_cast<float4 *>(spec + e0) = d_floor_mul(f0, r0);
    if (C == 2) {
        const float4 f1 = d_floor_quad(h.k1, h.c1, s_db, reinterpret_cast<const uint4 *>(tabs1), tabs1 + kSegStride * 16, words, 4 * q,
                                       dense, zero, e1);
        if (STREAM) __stcs(reinterpret_cast<float4 *>(spec + e1), d_floor_mul(f1, r1));
        else *reinterpret_cast<float4 *>(spec + e1) = d_floor_mul(f1, r1);
    }
}

// Persistent CTAs striding over the packets (grid = min(packets, a few CTAs per SM)).  Requires every coeff_off
// (and the arena bases) to be multiples of 4 elements, <= 8 channels, a uniform channel count C.
// Per packet: every global read the packet needs -- residue quads, the rows' segment tables and indices -- is issued
// at the top (one exposed memory latency), the tables land in shared memory, and the per-bin work runs out of it.
// VQ: the residue does not come from `residue` but from the packet's VQ records (d_vq_accumulate).
template <bool VQ>
__global__ void __launch_bounds__(kPfThreads, 4)
k_prologue_fused(const DevPacket *__restrict__ pkts, uint32_t n_pk, const float *__restrict__ residue, const float *__restrict__ dense_floor,
                 const float *__restrict__ zero_floor, const uint8_t *__restrict__ floor_kind, const uint4 *__restrict__ segtab, const uint8_t *__restrict__ seg_cnt,
                 const unsigned char *__restrict__ seg_index, int words, float *__restrict__ spec,
                 VqDev vq)
{
    extern __shared__ __align__(16) unsigned char pf_smem[];
    __shared__ float s_db[256];
    const int tid = threadIdx.x;
    s_db[tid] = c_inverse_db[tid];
    if (blockIdx.x >= n_pk) return;
    const int C = pkts[blockIdx.x].channels;                      // uniform over the batch
    const size_t ixs = seg_index_stride(words), rowb = pf_row_bytes(words);
    const int row_q = (int)(rowb >> 4), tab_q = kSegStride;       // 16-byte quads per row: table, then index
    float4 *s_r = reinterpret_cast<float4 *>(pf_smem + (size_t)C * rowb);     // [C][kPfThreads] when C > 1
    float *s_acc = reinterpret_cast<float *>(pf_smem + (size_t)C * rowb + (C > 1 ? (size_t)C * kPfThreads * sizeof(float4) : 0));   // VQ: [C][n2]
    if (!VQ && C <= 2) {
        // One or two channels, dense residue: the packets are software-pipelined.  While packet k is computed out of one
        // table buffer, everything packet k + 1 needs is already on its way: its rows' tables by cp.async into the other
        // buffer, its residue quads and header fields into registers.  One CTA barrier per packet.
        const int row_q2 = C * row_q;                                 // quads of one table buffer
        unsigned char *bufs[2] = {pf_smem, pf_smem + (size_t)C * rowb};
        const uint32_t bufs_s[2] = {smem_u32(bufs[0]), smem_u32(bufs[1])};
        auto prefetch = [&](uint32_t pk, int b, PfStereo &h, float4 &a0, float4 &a1) {
            const size_t row0 = (size_t)pk * C;
            for (int i = tid; i < row_q2; i += kPfThreads) {        // (one pass: <= 2 rows of <= 109 quads)
                const int c = i >= row_q ? 1 : 0, j = i - (c ? row_q : 0);
                const void *src = j < tab_q ? (const void *)(segtab + (row0 + c) * kSegStride + j)
                                            : (const void *)(reinterpret_cast<const uint4 *>(seg_index + (row0 + c) * ixs) + (j - tab_q));
                cp_async16(bufs_s[b] + 16u * (uint32_t)i, src);
            }
            cp_async_commit();
            const DevPacket &p = pkts[pk];
            h = d_pf_stereo_head(p, p.setup->mappings[p.mapping], C, floor_kind + p.pkt_index * C, seg_cnt + row0);
            a0 = make_float4(0.f, 0.f, 0.f, 0.f); a1 = a0;
            if (tid < (h.n2 >> 2)) {
                a0 = __ldcs(reinterpret_cast<const float4 *>(residue + h.base + 4 * (uint64_t)tid));
                if (C == 2) a1 = __ldcs(reinterpret_cast<const float4 *>(residue + h.base + h.n2 + 4 * (uint64_t)tid));
            }
        };
        PfStereo h, hn;
        float4 r0, r1, rn0, rn1;
        int b = 0;
        prefetch(blockIdx.x, 0, h, r0, r1);
        for (uint32_t pk = blockIdx.x; pk < n_pk; pk += gridDim.x, b ^= 1) {
            cp_async_wait<0>();
            __syncthreads();              // this packet's tables are in; everybody is done with the other buffer
            const uint32_t nx = pk + gridDim.x;
            if (nx < n_pk) prefetch(nx, b ^ 1, hn, rn0, rn1);
            const int n2 = h.n2;
            if (h.nsteps <= 1) {
                for (int q = tid; q < (n2 >> 2); q += kPfThreads) {
                    if (q != tid) {                               // blocks of more than 1024 bins: further passes
                        r0 = *reinterpret_cast<const float4 *>(residue + h.base + 4 * (uint64_t)q);
                        if (C == 2) r1 = *reinterpret_cast<const float4 *>(residue + h.base + n2 + 4 * (uint64_t)q);
                    }
                    d_pf_stereo_quad<true>(h, C, q, r0, r1, bufs[b], rowb, words, s_db, dense_floor, zero_floor, spec);
                }
            } else {
                // several coupling steps over two channels (legal, never seen): in order, one bin at a time
                const DevMapping &mp = pkts[pk].setup->mappings[pkts[pk].mapping];
                const uint4 *t0 = reinterpret_cast<const uint4 *>(bufs[b]), *t1 = reinterpret_cast<const uint4 *>(bufs[b] + rowb);
                const unsigned char *x0 = bufs[b] + (size_t)tab_q * 16, *x1 = x0 + rowb;
                for (int q = tid; q < (n2 >> 2); q += kPfThreads) {
                    const uint64_t e0 = h.base + 4 * (uint64_t)q, e1 = e0 + n2;
                    float4 v[2];
                    v[0] = *reinterpret_cast<const float4 *>(residue + e0);
                    v[1] = *reinterpret_cast<const float4 *>(residue + e1);
                    for (int s2 = h.nsteps - 1; s2 >= 0; s2--) d_inverse_couple(v[mp.mag[s2] & 1], v[mp.ang[s2] & 1]);
                    const float4 f0 = d_floor_quad(h.k0, h.c0, s_db, t0, x0, words, 4 * q, dense_floor, zero_floor, e0);
                    const float4 f1 = d_floor_quad(h.k1, h.c1, s_db, t1, x1, words, 4 * q, dense_floor, zero_floor, e1);
                    *reinterpret_cast<float4 *>(spec + e0) = d_floor_mul(f0, v[0]);
                    *reinterpret_cast<float4 *>(spec + e1) = d_floor_mul(f1, v[1]);
                }
            }
            h = hn; r0 = rn0; r1 = rn1;
        }
        return;
    }
    for (uint32_t pk = blockIdx.x; pk < n_pk; pk += gridDim.x) {
        const DevPacket &p = pkts[pk];
        const DevSetup &su = *p.setup;
        const DevMapping &mp = su.mappings[p.mapping];
        const int n2 = p.n >> 1, nsteps = mp.n_coupling;
        const uint8_t *kinds = floor_kind + p.pkt_index * C;
        const uint64_t base = p.coeff_off;
        const size_t row0 = (size_t)pk * C;
        __syncthreads();                                          // the previous packet is done with the shared tables
        for (int i = tid; i < C * row_q; i += kPfThreads) {
            const int c = i / row_q, j = i - c * row_q;
            const int cnt = seg_cnt[row0 + c] & 0x7f;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (j < tab_q) { if (j <= cnt && cnt) v = segtab[(row0 + c) * kSegStride + j]; }
            else if (cnt) v = reinterpret_cast<const uint4 *>(seg_index + (row0 + c) * ixs)[j - tab_q];
            reinterpret_cast<uint4 *>(pf_smem)[i] = v;
        }
        if (VQ) {
            const uint64_t o0 = vq.run_off[p.pkt_index], o1 = vq.run_off[p.pkt_index + 1];
            const uint64_t e0 = vq.ent_off[p.pkt_index], e1 = vq.ent_off[p.pkt_index + 1];
            d_vq_accumulate(s_acc, C, n2, su, mp, vq.runs + o0, (uint32_t)(o1 - o0), vq.entries + e0, (uint32_t)(e1 - e0), tid, kPfThreads);
        }
        __syncthreads();
        if (VQ && C <= 2 && nsteps <= 1) {                        // (dense residue of this shape: the pipelined loop above)
            const PfStereo h = d_pf_stereo_head(p, mp, C, kinds, seg_cnt + row0);
            for (int q = tid; q < (n2 >> 2); q += kPfThreads) {
                const float4 r0 = *reinterpret_cast<const float4 *>(s_acc + 4 * q);
                const float4 r1 = C == 2 ? *reinterpret_cast<const float4 *>(s_acc + n2 + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
                d_pf_stereo_quad<false>(h, C, q, r0, r1, pf_smem, rowb, words, s_db, dense_floor, zero_floor, spec);
            }
            continue;
        }
        // general case: the thread's quads of all channels sit in shared memory (dynamic channel indices of the
        // coupling steps without predicated register arrays); every thread touches only its own column
        for (int q = tid; q < (n2 >> 2); q += kPfThreads) {
            const uint64_t e = base + 4 * (uint64_t)q;
            for (int c = 0; c < C; c++)
                s_r[c * kPfThreads + tid] = VQ ? *reinterpret_cast<const float4 *>(s_acc + (size_t)c * n2 + 4 * q)
                                               : *reinterpret_cast<const float4 *>(residue + e + (uint64_t)c * n2);
            for (int s = nsteps - 1; s >= 0; s--) {                      // audio.rs:991-1002
                float4 m4 = s_r[mp.mag[s] * kPfThreads + tid], a4 = s_r[mp.ang[s] * kPfThreads + tid];
                d_inverse_couple(m4, a4);
                s_r[mp.mag[s] * kPfThreads + tid] = m4;
                s_r[mp.ang[s] * kPfThreads + tid] = a4;
            }
            for (int c = 0; c < C; c++) {
                const uint64_t ec = e + (uint64_t)c * n2;
                const float4 f = d_floor_quad(kinds[c], seg_cnt[row0 + c], s_db, reinterpret_cast<const uint4 *>(pf_smem + c * rowb),
                                              pf_smem + c * rowb + (size_t)tab_q * 16, words, 4 * q, dense_floor, zero_floor, ec);
                *reinterpret_cast<float4 *>(spec + ec) = d_floor_mul(f, s_r[c * kPfThreads + tid]);
            }
        }
    }
}

inline void prologue_kernel_configure()
{
    cudaFuncSetAttribute(k_floor1_segments, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)floor1_segments_smem(128));
    cudaFuncSetAttribute(k_prologue_fused<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prologue_fused_smem(8, kPfMaxWords));
    cudaFuncSetAttribute(k_prologue_fused<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)prologue_fused_smem(8, kPfMaxWords, kVqMaxElems));
}

}  // namespace lwb
