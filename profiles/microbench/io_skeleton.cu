// io_skeleton.cu -- how fast can the I/O pattern of k_long go with no arithmetic at all?
// Same structure: one CTA per SM x 12 warps, each warp streams 4 KB tiles by 1-D TMA into a 3-deep ring,
// reads them with 8 LDS.128 per lane and writes 4 KB of output with 32 STG.32 per lane, each a full
// 128-byte line (mode 0: k_long's scattered line order; mode 1: 8 coalesced STG.128 per lane).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o io_skeleton io_skeleton.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(c)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t b) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(b) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(384, 1) k_io(const float *__restrict__ in, float *__restrict__ out, uint32_t n_chains,
                                               uint32_t packets, unsigned int *ticket)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *tiles = reinterpret_cast<float *>(smem) + warp * 3 * 1024;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + 12 * 3 * 4096) + warp * 3;
    if (lane == 0) { for (int i = 0; i < 3; i++) mbar_init(smem_u32(&bars[i]), 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    uint32_t phase = 0;
    for (;;) {
        uint32_t c = 0;
        if (lane == 0) c = atomicAdd(ticket, 1u);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c >= n_chains) break;
        const float *src = in + (size_t)(c >> 1) * packets * 2048 + (c & 1) * 1024;      // stereo interleave like the bench
        float *dst = out + (size_t)c * packets * 1024;
        if (lane == 0)
            for (uint32_t i = 0; i < 3 && i < packets; i++) {
                mbar_expect_tx(smem_u32(&bars[i]), 4096);
                tma_load_1d(smem_u32(tiles + i * 1024), src + (size_t)i * 2048, 4096, smem_u32(&bars[i]));
            }
        uint32_t s = 0;
        for (uint32_t p = 0; p < packets; p++) {
            mbar_wait(smem_u32(&bars[s]), (phase >> s) & 1u);
            phase ^= 1u << s;
            const float4 *t4 = reinterpret_cast<const float4 *>(tiles + s * 1024);
            float4 q[8];
#pragma unroll
            for (int m = 0; m < 4; m++) { q[m] = t4[lane + 64 * m]; q[4 + m] = t4[63 - lane + 64 * m]; }
            __syncwarp();
            if (lane == 0 && p + 3 < packets) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar_expect_tx(smem_u32(&bars[s]), 4096);
                tma_load_1d(smem_u32(tiles + s * 1024), src + (size_t)(p + 3) * 2048, 4096, smem_u32(&bars[s]));
            }
            float *o = dst + (size_t)p * 1024;
            if (MODE == 0) {
                const float v[32] = {q[0].x, q[0].y, q[0].z, q[0].w, q[1].x, q[1].y, q[1].z, q[1].w, q[2].x, q[2].y, q[2].z, q[2].w,
                                     q[3].x, q[3].y, q[3].z, q[3].w, q[4].x, q[4].y, q[4].z, q[4].w, q[5].x, q[5].y, q[5].z, q[5].w,
                                     q[6].x, q[6].y, q[6].z, q[6].w, q[7].x, q[7].y, q[7].z, q[7].w};
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int r64 = 64 * (((j & 1) << 2) | (j & 2) | ((j >> 2) & 1));
                    __stcs(o + lane + r64, v[4 * j]);
                    __stcs(o + 63 - lane + r64, v[4 * j + 1]);
                    __stcs(o + 63 - lane + 960 - r64, v[4 * j + 2]);
                    __stcs(o + lane + 960 - r64, v[4 * j + 3]);
                }
            } else {
                float4 *o4 = reinterpret_cast<float4 *>(o);
#pragma unroll
                for (int m = 0; m < 8; m++) __stcs(o4 + lane + 32 * m, q[m]);
            }
            s = (s + 1 == 3) ? 0 : s + 1;
        }
    }
}

int main(int argc, char **argv)
{
    const uint32_t streams = 4096, packets = 16, chains = streams * 2;
    const size_t n = (size_t)chains * packets * 1024;
    float *in, *out;
    unsigned int *ticket;
    cudaMalloc(&in, n * 4); cudaMalloc(&out, n * 4); cudaMalloc(&ticket, 4096);
    cudaMemset(in, 0, n * 4);
    const size_t smem = 12 * 3 * 4096 + 12 * 3 * 8 + 64;
    cudaFuncSetAttribute(k_io<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(k_io<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int mode = 0; mode < 2; mode++) {
        float best = 1e9f;
        for (int it = 0; it < 12; it++) {
            cudaMemset(ticket, 0, 4);
            cudaEventRecord(e0);
            if (mode == 0) k_io<0><<<sms, 384, smem>>>(in, out, chains, packets, ticket);
            else k_io<1><<<sms, 384, smem>>>(in, out, chains, packets, ticket);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (it >= 2 && ms < best) best = ms;
        }
        printf("mode %d (%s): best %.3f ms  -> %.1f GB/s (read+write), err=%s\n", mode, mode ? "STG.128 coalesced" : "k_long line order STG.32",
               best, 2.0 * n * 4 / best / 1e6, cudaGetErrorString(cudaGetLastError()));
    }
    // plain device-to-device copy for reference
    float best = 1e9f;
    for (int it = 0; it < 8; it++) {
        cudaEventRecord(e0); cudaMemcpyAsync(out, in, n * 4, cudaMemcpyDeviceToDevice); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (it >= 2 && ms < best) best = ms;
    }
    printf("cudaMemcpy D2D: best %.3f ms -> %.1f GB/s\n", best, 2.0 * n * 4 / best / 1e6);
    return 0;
}
