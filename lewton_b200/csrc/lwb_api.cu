// lwb_api.cu -- the C ABI (include/lewton_b200.h): context, setup, stream state and batch
// submission.  Host logic mirrors the control flow of lewton's read_audio_packet_generic back
// half (src/audio.rs:988-1157): which window shape a packet has, whether a previous right half
// exists, what the packet returns -- all of that is decided here on the host from the mode bits
// (it never depends on sample values), so the kernels receive fully resolved descriptors and the
// device never has to be synchronised to learn a length.
#include <cuda_runtime.h>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <new>
#include <string>
#include <vector>

#include "kernel_long.cuh"
#include "kernel_short.cuh"
#include "kernel_mid.cuh"
#include "kernels_generic.cuh"
#include "kernel_chain.cuh"
#include "kernel_prologue.cuh"
#include "kernel_floor0.cuh"
#include "lwb_common.h"
#include "pcm_copy_plan.h"
#include "../../include/lewton_frontend.h"
#include "batcher.h"

namespace lwb {
int generate_tables(int bs, float *a, float *b, float *c, float *window, uint32_t *bitrev);
int prepare_floor1(const lwb_floor_desc &d, DevFloor1 *out);
}  // namespace lwb
namespace lwf {
std::vector<float> bark_map_cos_omega(uint16_t n, uint16_t rate, uint16_t bark_map_size);   // frontend.cpp
void floor0_descs(const lwf_headers *h, std::vector<uint32_t> *index, std::vector<lwb_floor0_desc> *descs);
}  // namespace lwf

using namespace lwb;

#include "host_objects.cuh"

// ---------------------------------------------------------------------------------------------
// library / context
// ---------------------------------------------------------------------------------------------
extern "C" int lwb_abi_version(void) { return LWB_ABI_VERSION; }

extern "C" int lwb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int lwb_ctx_create(int device, lwb_ctx **out)
{
    if (!out) return LWB_ERR_INVALID;
    *out = nullptr;
    int n = lwb_device_count();
    if (n <= 0 || device < 0 || device >= n) return LWB_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return LWB_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return LWB_ERR_NO_DEVICE;   // kernels are built for sm_90a only
    lwb_ctx *ctx = new (std::nothrow) lwb_ctx();
    if (!ctx) return LWB_ERR_BUFFER;
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaSetDevice(device) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx;
        return LWB_ERR_CUDA;
    }
    if (create_pipeline_objects(ctx)) {
        lwb_ctx_destroy(ctx);
        return LWB_ERR_CUDA;
    }
    if (const char *e = getenv("LWB_SCRATCH_MB")) {
        long mb = atol(e);
        if (mb >= 1) ctx->x_cap_elems = (size_t)mb << 18;
    }
    long_kernel_configure();
    short_kernel_configure();
    mid_kernel_configure();
    prologue_kernel_configure();
    *out = ctx;
    return LWB_OK;
}

// The compute stream and both copy streams: a host-memory batch's last D2H may still run after its kernels.
static cudaError_t sync_all_streams(lwb_ctx *ctx)
{
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    for (cudaStream_t s : {ctx->copy_in, ctx->copy_out}) {
        const cudaError_t e2 = s ? cudaStreamSynchronize(s) : cudaSuccess;
        if (e == cudaSuccess) e = e2;
    }
    return e;
}

extern "C" void lwb_ctx_destroy(lwb_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    sync_all_streams(ctx);
    for (DevBuf *b : {&ctx->spec, &ctx->segtab, &ctx->magic, &ctx->x, &ctx->desc, &ctx->chains, &ctx->ticket, &ctx->runs_buf[0],
                      &ctx->runs_buf[1], &ctx->cdesc, &ctx->cbytes, &ctx->floor0, &ctx->state_rows, &ctx->win})
        if (b->p) cudaFree(b->p);
    auto free_set = [](ArenaSet &s) {
        for (DevBuf *b : {&s.coeffs, &s.dense, &s.pcm, &s.kinds, &s.ys, &s.vqoff, &s.vqrec})
            if (b->p) cudaFree(b->p);
        if (s.done) cudaEventDestroy(s.done);
    };
    for (ArenaSet &s : ctx->host_sets) free_set(s);
    free_set(ctx->ordered);
    for (cudaEvent_t e : ctx->ticket_events) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->spare_events) cudaEventDestroy(e);
    for (CachedTables &ct : ctx->tables)
        for (void *p : ct.allocs) cudaFree(p);
    for (void *h : ctx->stage_old) cudaFreeHost(h);
    for (Staging &st : ctx->stage) {
        if (st.h) cudaFreeHost(st.h);
        if (st.ev) cudaEventDestroy(st.ev);
    }
    for (cudaEvent_t e : ctx->ev_in) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->ev_done) if (e) cudaEventDestroy(e);
    for (int k = 0; k < 2; k++) {
        if (ctx->ev_desc[k]) cudaEventDestroy(ctx->ev_desc[k]);
        if (ctx->ev_kdone[k]) cudaEventDestroy(ctx->ev_kdone[k]);
    }
    cudaStreamDestroy(ctx->stream);
    cudaStreamDestroy(ctx->copy_in);
    cudaStreamDestroy(ctx->copy_out);
    delete ctx;
}

extern "C" int lwb_ctx_synchronize(lwb_ctx *ctx)
{
    if (!ctx) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, sync_all_streams(ctx));
    return retire_tickets(ctx, ctx->tickets_issued, true);
}

extern "C" const char *lwb_last_error(const lwb_ctx *ctx) { return ctx ? ctx->err.c_str() : "no context"; }
extern "C" void *lwb_ctx_cuda_stream(lwb_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }
extern "C" uint64_t lwb_ctx_launch_count(const lwb_ctx *ctx) { return ctx ? ctx->launches : 0; }
extern "C" uint64_t lwb_ctx_kernel_launches(const lwb_ctx *ctx, int kernel_id)
{
    return ctx && kernel_id >= 0 && kernel_id < LWB_KERNEL_COUNT ? ctx->kernel_launches[kernel_id] : 0;
}

extern "C" void *lwb_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
extern "C" void lwb_host_free(void *p) { if (p) cudaFreeHost(p); }

// NUMA placement of the host side.  A rank that feeds GPU d through host buffers should run on, and
// allocate its pinned memory from, the socket GPU d's PCIe root hangs off: with 4 GPUs per socket the
// copies of all of them otherwise cross the inter-socket link of whichever node the pages landed on.
// Plain syscalls (no libnuma dependency).  Returns the node, or -1 when it cannot be determined.
extern "C" int lwb_bind_host_to_device(int device)
{
    if (device < 0) {
        syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
        return -1;
    }
    char busid[64] = {0};
    if (cudaDeviceGetPCIBusId(busid, (int)sizeof(busid) - 1, device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char *c = busid; *c; c++) *c = (char)tolower((unsigned char)*c);
    char path[160];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", busid);
    int node = -1;
    if (FILE *f = fopen(path, "r")) {
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
    }
    if (node < 0 || node >= 1024) return -1;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    cpu_set_t want, cur;
    CPU_ZERO(&want);
    if (FILE *f = fopen(path, "r")) {
        int a, b;
        while (fscanf(f, "%d", &a) == 1) {
            b = a;
            int ch = fgetc(f);
            if (ch == '-') {
                if (fscanf(f, "%d", &b) != 1) break;
                ch = fgetc(f);
            }
            for (int k = a; k <= b && k < CPU_SETSIZE; k++) CPU_SET(k, &want);
            if (ch != ',') break;
        }
        fclose(f);
    }
    if (sched_getaffinity(0, sizeof(cur), &cur) == 0) {
        cpu_set_t both;
        CPU_AND(&both, &want, &cur);
        if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof(both), &both);
    }
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, (unsigned long)(sizeof(mask) * 8));
    return node;
}

extern "C" int lwb_device_alloc(lwb_ctx *ctx, size_t bytes, void **out)
{
    if (!ctx || !out) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, cudaMalloc(out, bytes ? bytes : 1));
    return LWB_OK;
}
extern "C" void lwb_device_free(lwb_ctx *ctx, void *p)
{
    if (!ctx || !p) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaFree(p);
}
extern "C" int lwb_memcpy_h2d(lwb_ctx *ctx, void *dst, const void *src, size_t bytes)
{
    if (!ctx) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LWB_OK;
}
extern "C" int lwb_memcpy_d2h(lwb_ctx *ctx, void *dst, const void *src, size_t bytes)
{
    if (!ctx) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LWB_OK;
}

extern "C" int lwb_tables_generate(int bs, float *a, float *b, float *c, float *window, uint32_t *bitrev)
{
    return generate_tables(bs, a, b, c, window, bitrev);
}

// ---------------------------------------------------------------------------------------------
// setup
// ---------------------------------------------------------------------------------------------
template <typename T>
static int upload(lwb_setup *su, const T *host, size_t count, const T **dev)
{
    void *p = nullptr;
    lwb_ctx *ctx = su->ctx;
    CU(ctx, cudaMalloc(&p, std::max<size_t>(count * sizeof(T), 16)));
    su->allocs.push_back(p);
    if (count) CU(ctx, cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    *dev = (const T *)p;
    return LWB_OK;
}

extern "C" void lwb_setup_destroy(lwb_setup *su)
{
    if (!su) return;
    cudaSetDevice(su->ctx->device);
    cudaStreamSynchronize(su->ctx->stream);
    for (void *p : su->allocs) cudaFree(p);
    delete su;
}

extern "C" int lwb_setup_create(lwb_ctx *ctx, const lwb_setup_desc *d, lwb_setup **out)
{
    if (!ctx || !d || !out) return LWB_ERR_INVALID;
    *out = nullptr;
    // header.rs:239-243 (blocksizes, channels)
    if (d->blocksize_0 < 6 || d->blocksize_0 > 13 || d->blocksize_1 < 6 || d->blocksize_1 > 13 ||
        d->blocksize_0 > d->blocksize_1 || d->audio_channels == 0)
        return fail(ctx, LWB_ERR_BAD_FORMAT, "setup: blocksizes/channels out of range");
    if (d->n_modes == 0 || d->n_modes > LWB_MAX_MODES || d->n_mappings == 0 || d->n_mappings > 64 ||
        d->n_floors == 0 || d->n_floors > 64 || !d->modes || !d->mappings || !d->floors)
        return fail(ctx, LWB_ERR_INVALID, "setup: counts out of range");
    // A caller's bit-reversal table must be compute_bitreverse(bs) (header_cached.rs:101-110), the only one the crate
    // makes: k_long, k_mid and k_short build that permutation into their index maps, so any other table would give PCM
    // that depends on the batch path.
    for (int i = 0; i < 2; i++) {
        const lwb_tables_ref &t = d->tables[i];
        if (!t.a || !t.bitrev) continue;
        const int bs = i ? d->blocksize_1 : d->blocksize_0;
        std::vector<uint32_t> br(((size_t)1 << bs) / 8);
        generate_tables(bs, nullptr, nullptr, nullptr, nullptr, br.data());
        if (!std::equal(br.begin(), br.end(), t.bitrev))
            return fail(ctx, LWB_ERR_INVALID, i ? "setup: tables[1].bitrev is not compute_bitreverse(blocksize_1)"
                                                : "setup: tables[0].bitrev is not compute_bitreverse(blocksize_0)");
    }
    CU(ctx, cudaSetDevice(ctx->device));
    lwb_setup *su = new (std::nothrow) lwb_setup();
    if (!su) return LWB_ERR_BUFFER;
    su->ctx = ctx;
    su->channels = d->audio_channels;
    su->bs0 = d->blocksize_0;
    su->bs1 = d->blocksize_1;
    su->n_modes = d->n_modes;
    su->n_mappings = d->n_mappings;
    std::memset(&su->host, 0, sizeof(su->host));
    int rc = LWB_OK;
    // tables (header_cached.rs:33-41): the caller's own, or generated here
    for (int i = 0; i < 2 && rc == LWB_OK; i++) {
        const int bs = i ? d->blocksize_1 : d->blocksize_0;
        const size_t n = (size_t)1 << bs;
        std::vector<float> a(n / 2), b(n / 2), c(n / 4), w(n / 2);
        std::vector<uint32_t> br(n / 8);
        const lwb_tables_ref &t = d->tables[i];
        if (t.a) {
            if (!t.b || !t.c || !t.window || !t.bitrev) { rc = LWB_ERR_INVALID; break; }
            std::copy(t.a, t.a + n / 2, a.begin());
            std::copy(t.b, t.b + n / 2, b.begin());
            std::copy(t.c, t.c + n / 4, c.begin());
            std::copy(t.window, t.window + n / 2, w.begin());
            std::copy(t.bitrev, t.bitrev + n / 8, br.begin());
        } else {
            generate_tables(bs, a.data(), b.data(), c.data(), w.data(), br.data());
        }
        // Blocksize tables live in the context and are shared by every setup that has the same ones (bit for
        // bit): streams opened from different headers then still run in one launch of the fused kernels, which
        // take one twiddle pack per launch.
        const CachedTables *hit = nullptr;
        for (const CachedTables &ct : ctx->tables)
            if (ct.dt.bs == bs && ct.a == a && ct.b == b && ct.c == c && ct.w == w && ct.br == br) { hit = &ct; break; }
        if (!hit) {
            CachedTables ct;
            ct.dt.bs = bs;
            ct.dt.pad = 0;
            ct.dt.pack = nullptr;
            auto up = [&](const void *h, size_t bytes, const void **dev) {
                void *p = nullptr;
                if (cudaMalloc(&p, std::max<size_t>(bytes, 16)) != cudaSuccess) return LWB_ERR_CUDA;
                ct.allocs.push_back(p);
                if (cudaMemcpyAsync(p, h, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return LWB_ERR_CUDA;
                *dev = p;
                return LWB_OK;
            };
            std::vector<float> pack;
            if (bs == kLongBs) {
                pack.resize(kLongPackFloats);
                long_build_pack(a.data(), b.data(), c.data(), w.data(), pack.data());
            } else if (bs == kShortBs) {
                pack.resize(kShortPackFloats);
                short_build_pack(a.data(), b.data(), c.data(), w.data(), pack.data());
            } else if (bs == 10) {
                pack.resize(kLongPackFloats);
                mid_build_pack<1>(a.data(), b.data(), c.data(), w.data(), pack.data());
            } else if (bs == 9) {
                pack.resize(kLongPackFloats);
                mid_build_pack<2>(a.data(), b.data(), c.data(), w.data(), pack.data());
            }
            rc = up(a.data(), a.size() * 4, (const void **)&ct.dt.a);
            if (!rc) rc = up(b.data(), b.size() * 4, (const void **)&ct.dt.b);
            if (!rc) rc = up(c.data(), c.size() * 4, (const void **)&ct.dt.c);
            if (!rc) rc = up(w.data(), w.size() * 4, (const void **)&ct.dt.window);
            if (!rc) rc = up(br.data(), br.size() * 4, (const void **)&ct.dt.bitrev);
            if (!rc && !pack.empty()) rc = up(pack.data(), pack.size() * 4, (const void **)&ct.dt.pack);
            // the copies above read from vectors that die here
            if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = LWB_ERR_CUDA;
            if (rc) {
                for (void *p : ct.allocs) cudaFree(p);
                fail(ctx, rc, "setup: table upload");
                break;
            }
            ct.a = a; ct.b = b; ct.c = c; ct.w = w; ct.br = br;
            ctx->tables.push_back(std::move(ct));
            hit = &ctx->tables.back();
        }
        su->host.tab[i] = hit->dt;
    }
    std::vector<DevFloor1> floors(d->n_floors);
    for (uint32_t i = 0; i < d->n_floors && rc == LWB_OK; i++) rc = prepare_floor1(d->floors[i], &floors[i]);
    for (uint32_t i = 0; i < d->n_floors; i++) su->floor_types.push_back(d->floors[i].floor_type);
    su->mappings.resize(d->n_mappings);
    for (uint32_t i = 0; i < d->n_mappings && rc == LWB_OK; i++) {
        const lwb_mapping_desc &m = d->mappings[i];
        DevMapping &dm = su->mappings[i];
        std::memset(&dm, 0, sizeof(dm));
        if (m.coupling_steps > LWB_MAX_COUPLING || m.submaps == 0 || m.submaps > LWB_MAX_SUBMAPS) {
            rc = LWB_ERR_BAD_FORMAT;
            break;
        }
        dm.n_coupling = m.coupling_steps;
        for (int s = 0; s < m.coupling_steps; s++) {
            // header.rs:1006-1011
            if (m.magnitudes[s] == m.angles[s] || m.magnitudes[s] >= d->audio_channels ||
                m.angles[s] >= d->audio_channels) {
                rc = LWB_ERR_BAD_FORMAT;
                break;
            }
            dm.mag[s] = m.magnitudes[s];
            dm.ang[s] = m.angles[s];
        }
        for (int c = 0; c < d->audio_channels && rc == LWB_OK; c++) {
            if (m.mux[c] >= m.submaps || m.submap_floors[m.mux[c]] >= d->n_floors) {
                rc = LWB_ERR_BAD_FORMAT;      // header.rs:1023-1026, 1043-1047
                break;
            }
            dm.floor_of_channel[c] = m.submap_floors[m.mux[c]];
            if (d->audio_channels <= 8) dm.sub_ch[m.mux[c]][dm.sub_nch[m.mux[c]]++] = (uint8_t)c;
        }
    }
    for (uint32_t i = 0; i < d->n_modes && rc == LWB_OK; i++) {
        if (d->modes[i].mapping >= d->n_mappings) { rc = LWB_ERR_BAD_FORMAT; break; }   // header.rs:1067-1072
        su->host.mode_blockflag[i] = d->modes[i].blockflag ? 1 : 0;
        su->host.mode_mapping[i] = d->modes[i].mapping;
    }
    // LWB_ENTRY_VQ: codebook value tables and residue partition sizes
    if (rc == LWB_OK && d->n_codebooks) {
        if (d->n_codebooks > 256 || !d->codebooks || d->n_residues > (uint32_t)kMaxResidues || (d->n_residues && !d->residues)) {
            rc = LWB_ERR_INVALID;
        } else {
            std::vector<DevBook> books(d->n_codebooks);
            for (uint32_t i = 0; i < d->n_codebooks && rc == LWB_OK; i++) {
                const lwb_codebook_desc &cb = d->codebooks[i];
                books[i].vq = nullptr;
                books[i].entries = cb.entries;
                books[i].dims = cb.dimensions;
                books[i].pad = 0;
                if (cb.vq && cb.entries && cb.dimensions) rc = upload(su, cb.vq, (size_t)cb.entries * cb.dimensions, &books[i].vq);
            }
            if (rc == LWB_OK) rc = upload(su, books.data(), books.size(), &su->host.books);
            // (the uploads read the caller's tables: done before we return, see the synchronise below)
            if (rc == LWB_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = LWB_ERR_CUDA;
            su->host.n_books = d->n_codebooks;
            su->host.n_residues = d->n_residues;
            for (uint32_t i = 0; i < d->n_residues; i++) su->host.res_psize[i] = d->residues[i].partition_size;
        }
    }
    if (rc == LWB_OK) rc = upload(su, floors.data(), floors.size(), &su->host.floors);
    if (rc == LWB_OK) rc = upload(su, su->mappings.data(), su->mappings.size(), &su->host.mappings);
    su->host.channels = d->audio_channels;
    su->host.bs0 = d->blocksize_0;
    su->host.bs1 = d->blocksize_1;
    su->host.n_floors = (uint8_t)d->n_floors;
    if (rc == LWB_OK) {
        const DevSetup *dp = nullptr;
        rc = upload(su, &su->host, 1, &dp);
        su->d_setup = const_cast<DevSetup *>(dp);
    }
    if (rc == LWB_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = LWB_ERR_CUDA;
    if (rc != LWB_OK) {
        lwb_setup_destroy(su);
        if (ctx->err.empty() || rc != LWB_ERR_CUDA) ctx->err = "setup: rejected (see header.rs validation rules)";
        return rc;
    }
    *out = su;
    return LWB_OK;
}

extern "C" int lwb_setup_set_floor0(lwb_setup *su, uint32_t fi, const lwb_floor0_desc *d)
{
    if (!su || !d) return LWB_ERR_INVALID;
    lwb_ctx *ctx = su->ctx;
    if (fi >= su->floor_types.size() || su->floor_types[fi] != LWB_FLOOR_TYPE_ZERO)
        return fail(ctx, LWB_ERR_INVALID, "set_floor0: no type-0 floor at that index");
    if (d->order < 2 || d->order > LWB_MAX_POSTS - 2 || d->amplitude_bits < 1 || d->amplitude_bits > 64 || !d->rate || !d->bark_map_size)
        return fail(ctx, LWB_ERR_INVALID, "set_floor0: order must be 2..63, amplitude_bits 1..64, rate and bark_map_size nonzero");
    // Streams (and the batches and plans built on them) read the setup's description as it was: it is fixed from then on.
    if (su->streams_opened) return fail(ctx, LWB_ERR_INVALID, "set_floor0: the setup already has streams");
    CU(ctx, cudaSetDevice(ctx->device));
    // a floor described again: its earlier tables and the earlier description array go
    auto release = [&](const void *p) {
        auto it = std::find(su->allocs.begin(), su->allocs.end(), p);
        if (p && it != su->allocs.end()) {
            cudaFree(*it);
            su->allocs.erase(it);
        }
    };
    DevFloor0 f;
    std::memset(&f, 0, sizeof(f));
    f.order = d->order;
    f.amplitude_offset = d->amplitude_offset;
    f.max_amp = d_floor0_max_amp(d->amplitude_bits);
    for (int i = 0; i < 2; i++) {
        const uint16_t n2 = (uint16_t)(1u << ((i ? su->bs1 : su->bs0) - 1));
        std::vector<float> bark = d->bark_cos_omega[i] ? std::vector<float>(d->bark_cos_omega[i], d->bark_cos_omega[i] + n2)
                                                       : lwf::bark_map_cos_omega(n2, d->rate, d->bark_map_size);
        int rc = upload(su, bark.data(), bark.size(), &f.bark_cos_omega[i]);
        if (rc) return rc;
        CU(ctx, cudaStreamSynchronize(ctx->stream));              // (the copy reads `bark`)
    }
    if (su->floor0.empty()) su->floor0.assign(su->floor_types.size(), DevFloor0{});
    release(su->floor0[fi].bark_cos_omega[0]);
    release(su->floor0[fi].bark_cos_omega[1]);
    release(su->host.floor0);
    su->floor0[fi] = f;
    const DevFloor0 *dev = nullptr;
    int rc = upload(su, su->floor0.data(), su->floor0.size(), &dev);
    if (rc) return rc;
    su->host.floor0 = dev;
    CU(ctx, cudaMemcpyAsync(su->d_setup, &su->host, sizeof(su->host), cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LWB_OK;
}

extern "C" int lwb_setup_set_output_mix(lwb_setup *su, uint32_t n_out, const float *m)
{
    if (!su) return LWB_ERR_INVALID;
    lwb_ctx *ctx = su->ctx;
    const unsigned C = su->channels;
    if ((n_out == 0) != (m == nullptr) || n_out > 8) return fail(ctx, LWB_ERR_INVALID, "set_output_mix: n_out must be 1..8 with a matrix, or 0 with none");
    for (size_t i = 0; i < (size_t)n_out * C; i++)
        if (!std::isfinite(m[i])) return fail(ctx, LWB_ERR_INVALID, "set_output_mix: a coefficient is not finite");
    // Streams (and the batches and plans built on them) lay out their PCM by the setup's output channels: fixed from then on.
    if (su->streams_opened) return fail(ctx, LWB_ERR_INVALID, "set_output_mix: the setup already has streams");
    CU(ctx, cudaSetDevice(ctx->device));
    // per output row, its nonzero coefficients in ascending channel order
    std::vector<uint8_t> ch;
    std::vector<float> w;
    DevSetup h = su->host;
    h.mix_ch = nullptr;
    h.mix_w = nullptr;
    std::memset(h.mix_row, 0, sizeof(h.mix_row));
    h.n_out = (uint8_t)n_out;
    for (uint32_t k = 0; k < n_out; k++) {
        for (unsigned c = 0; c < C; c++)
            if (m[(size_t)k * C + c] != 0.f) {
                ch.push_back((uint8_t)c);
                w.push_back(m[(size_t)k * C + c]);
            }
        h.mix_row[k + 1] = (uint16_t)ch.size();
    }
    for (uint32_t k = n_out; k < 8; k++) h.mix_row[k + 1] = h.mix_row[n_out];
    int rc;
    if (n_out && ((rc = upload(su, ch.data(), ch.size(), &h.mix_ch)) || (rc = upload(su, w.data(), w.size(), &h.mix_w)))) return rc;
    CU(ctx, cudaMemcpyAsync(su->d_setup, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));           // (the copies read `ch`, `w` and `h`)
    // the previous mix's term lists go
    for (const void *p : {(const void *)su->host.mix_ch, (const void *)su->host.mix_w}) {
        auto it = std::find(su->allocs.begin(), su->allocs.end(), p);
        if (p && it != su->allocs.end()) {
            cudaFree(*it);
            su->allocs.erase(it);
        }
    }
    su->host = h;
    return LWB_OK;
}

extern "C" uint32_t lwb_setup_output_channels(const lwb_setup *su) { return su ? su->out_channels() : 0; }

// The front half's setup with its record-capable type-0 floors described (here, beside lwb_setup_set_floor0: the front
// half alone builds without the synthesis library).
extern "C" int lwf_headers_make_setup_floor0(const lwf_headers *h, lwb_ctx *ctx, lwb_setup **out)
{
    int rc = lwf_headers_make_setup(h, ctx, out);
    if (rc) return rc;
    std::vector<uint32_t> index;
    std::vector<lwb_floor0_desc> descs;
    try {
        lwf::floor0_descs(h, &index, &descs);
    } catch (...) {
        rc = LWB_ERR_BUFFER;
    }
    for (size_t i = 0; i < descs.size() && !rc; i++) rc = lwb_setup_set_floor0(*out, index[i], &descs[i]);
    if (rc) {
        lwb_setup_destroy(*out);
        *out = nullptr;
    }
    return rc;
}

// ---------------------------------------------------------------------------------------------
// stream state
// ---------------------------------------------------------------------------------------------
static size_t state_stride(const lwb_setup *su) { return (size_t)1 << (su->bs1 - 1); }

extern "C" int lwb_stream_open(lwb_ctx *ctx, const lwb_setup *su, lwb_stream **out)
{
    if (!ctx || !su || !out || su->ctx != ctx) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    lwb_stream *s = new (std::nothrow) lwb_stream();
    if (!s) return LWB_ERR_BUFFER;
    su->streams_opened = true;
    s->ctx = ctx;
    s->setup = su;
    cudaError_t e = cudaMalloc((void **)&s->d_state, su->channels * state_stride(su) * sizeof(float));
    if (e != cudaSuccess) {
        delete s;
        return fail(ctx, LWB_ERR_CUDA, "stream_open: cudaMalloc", e);
    }
    *out = s;
    return LWB_OK;
}

extern "C" void lwb_stream_destroy(lwb_stream *s)
{
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    sync_all_streams(s->ctx);
    cudaFree(s->d_state);
    delete s;
}

extern "C" int lwb_stream_reset(lwb_stream *s)
{
    if (!s) return LWB_ERR_INVALID;
    set_stream_state(s, false, 0);
    return LWB_OK;
}
extern "C" int lwb_stream_set_window(lwb_stream *s, uint64_t skip, uint64_t limit)
{
    if (!s) return LWB_ERR_INVALID;
    s->skip_left = skip;
    s->limit_left = limit;
    s->ctx->windows_set = true;
    s->ctx->state_gen++;           // prepared batches holding the stream plan again
    return LWB_OK;
}
extern "C" int lwb_stream_window(const lwb_stream *s, uint64_t *skip_left, uint64_t *limit_left)
{
    if (!s) return LWB_ERR_INVALID;
    if (skip_left) *skip_left = s->skip_left;
    if (limit_left) *limit_left = s->limit_left;
    return LWB_OK;
}
extern "C" int lwb_stream_is_empty(const lwb_stream *s) { return (!s || !s->has) ? 1 : 0; }
extern "C" uint32_t lwb_stream_state_len(const lwb_stream *s) { return (s && s->has) ? s->plen : 0; }

extern "C" int lwb_stream_clone(const lwb_stream *s, lwb_stream **out)
{
    if (!s || !out) return LWB_ERR_INVALID;
    int rc = lwb_stream_open(s->ctx, s->setup, out);
    if (rc) return rc;
    (*out)->has = s->has;
    (*out)->plen = s->plen;
    (*out)->skip_left = s->skip_left;
    (*out)->limit_left = s->limit_left;
    lwb_ctx *ctx = s->ctx;
    CU(ctx, cudaMemcpyAsync((*out)->d_state, s->d_state,
                            s->setup->channels * state_stride(s->setup) * sizeof(float),
                            cudaMemcpyDeviceToDevice, ctx->stream));
    return LWB_OK;
}

extern "C" int lwb_stream_export_state(lwb_stream *s, float *out)
{
    if (!s || !out) return LWB_ERR_INVALID;
    if (!s->has) return LWB_OK;
    lwb_ctx *ctx = s->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, cudaMemcpy2DAsync(out, s->plen * sizeof(float), s->d_state, state_stride(s->setup) * sizeof(float),
                              s->plen * sizeof(float), s->setup->channels, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LWB_OK;
}

extern "C" int lwb_stream_import_state(lwb_stream *s, const float *data, uint32_t len)
{
    if (!s || (!data && len)) return LWB_ERR_INVALID;
    if (len > state_stride(s->setup)) return LWB_ERR_BUFFER;
    lwb_ctx *ctx = s->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    if (len) {
        CU(ctx, cudaMemcpy2DAsync(s->d_state, state_stride(s->setup) * sizeof(float), data, len * sizeof(float),
                                  len * sizeof(float), s->setup->channels, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
    }
    s->ctx->state_gen++;           // contents changed even if the shape did not
    s->has = true;
    s->plen = len;
    return LWB_OK;
}

extern "C" int lwb_decoded_sample_count(const lwb_setup *su, uint8_t mode, int prev_flag, int next_flag,
                                        uint32_t *n_samples)
{
    if (!su || !n_samples) return LWB_ERR_INVALID;
    Geom g;
    int rc = geometry(su, mode, prev_flag, next_flag, &g);
    if (rc) return rc;
    *n_samples = g.rs - g.ls;
    return LWB_OK;
}

#include "path_generic.cuh"
#include "path_long.cuh"
#include "path_chain.cuh"
#include "path_mixed.cuh"
#include "path_mid.cuh"

// The batch paths in the order they are tried.  The last, the four-kernel path, takes every batch that reaches it.
using BatchPath = int (*)(lwb_ctx *, const lwb_chain *, size_t, const lwb_batch_io *, const BatchWalk &, bool *, lwb_plan *);
static constexpr BatchPath kBatchPaths[] = {try_long, try_mid, try_mixed, try_chain, try_generic};
constexpr size_t kChainPath = 3, kGenericPath = 4;
static_assert(kBatchPaths[kChainPath] == try_chain && kBatchPaths[kGenericPath] == try_generic && std::size(kBatchPaths) == kGenericPath + 1,
              "kChainPath / kGenericPath name the chain-kernel and the four-kernel path, the last one");

// Index of the first batch path to try.  LWB_FORCE_GENERIC is a test switch that sends batches to the reference
// paths: "1" to the four-kernel path only, any other value to the chain kernel and then the four-kernel path.
static size_t first_batch_path()
{
    const char *fg = getenv("LWB_FORCE_GENERIC");
    if (!fg) return 0;
    return std::strcmp(fg, "1") == 0 ? kGenericPath : kChainPath;
}

// The argument checks of a batch and what every path relies on: valid chains, each stream in one chain, and the residue
// entries' floor kinds and single channel count.
static int check_batch_args(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io)
{
    if (io->entry != LWB_ENTRY_SPECTRUM && io->entry != LWB_ENTRY_RESIDUE && io->entry != LWB_ENTRY_VQ) return fail(ctx, LWB_ERR_INVALID, "bad entry");
    if (io->memory != LWB_MEM_HOST && io->memory != LWB_MEM_DEVICE) return fail(ctx, LWB_ERR_INVALID, "bad memory space");
    if (!out_format_known(io->out_format)) return fail(ctx, LWB_ERR_INVALID, "bad out_format");
    if (n_chains == 0) return LWB_OK;
    if ((!io->coeffs && io->entry != LWB_ENTRY_VQ) || !io->pcm) return fail(ctx, LWB_ERR_INVALID, "null arena");
    if (io->entry == LWB_ENTRY_VQ && (!io->vq_runs || !io->vq_run_offsets || !io->vq_entries || !io->vq_entry_offsets || !io->floor_kind))
        return fail(ctx, LWB_ERR_INVALID, "VQ entry needs vq_runs, vq_entries, their offsets and floor_kind");
    const uint64_t epoch = ++ctx->epoch;      // per context: concurrent calls on different contexts share nothing
    const unsigned C = chains[0].stream ? chains[0].stream->setup->channels : 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        if (!c->stream || c->stream->ctx != ctx || (c->n_packets && !c->mode_numbers))
            return fail(ctx, LWB_ERR_INVALID, "chain: bad stream or mode list");
        if (c->stream->busy_epoch == epoch) return fail(ctx, LWB_ERR_INVALID, "a stream appears in two chains of one batch");
        c->stream->busy_epoch = epoch;
        if (io->entry != LWB_ENTRY_SPECTRUM) {
            if (c->stream->setup->channels != C) return fail(ctx, LWB_ERR_INVALID, "residue batches need one channel count");
            if (!io->floor_kind) return fail(ctx, LWB_ERR_INVALID, "residue entry needs floor_kind");
        }
    }
    return LWB_OK;
}

// Whether the ranges chain c's walk w touches end inside the 64-bit address space, in bytes: its PCM write set (the
// samples it writes, w.written), its
// coefficient (and dense floor) elements and, for the residue entries, its packet rows of floor1_y, the widest per-row
// array.  BatchExtent::add and the run descriptors sum these offsets in uint64_t; an offset near 2^64 would wrap to a
// small one and address memory the caller never named.
static bool chain_ranges_fit(const lwb_batch_io *io, const lwb_chain *c, const ChainWalk &w)
{
    const lwb_setup *su = c->stream->setup;
    const uint64_t K = su->out_channels(), esz = out_format_of(io->out_format).esz;
    uint64_t span, end;
    if (out_format_of(io->out_format).planar) {
        if (__builtin_mul_overflow(K - 1, c->out_stride, &span) || __builtin_add_overflow(span, w.written, &span)) return false;
    } else if (__builtin_mul_overflow(w.written, K, &span)) {
        return false;
    }
    if (__builtin_add_overflow(c->out_offset, span, &end) || __builtin_mul_overflow(end, esz, &end)) return false;
    // walk_chain sums the packets' C * n/2 (below 2^52) onto coeff_offset: coeff_end is below it exactly when that wrapped
    if (w.coeff_end < c->coeff_offset || __builtin_mul_overflow(w.coeff_end, (uint64_t)sizeof(float), &end)) return false;
    if (io->entry == LWB_ENTRY_SPECTRUM) return true;
    return !__builtin_add_overflow(c->packet_index, (uint64_t)w.done, &end) &&
           !__builtin_mul_overflow(end, (uint64_t)su->channels * LWB_MAX_POSTS * sizeof(uint32_t), &end);
}

// The one walk of a batch, made before a path is chosen: the argument checks, every chain's walk and the batch's extent,
// and every refusal a batch gets from its arguments and arrays -- an out_stride below the samples a chain writes,
// a chain range that does not fit in 64 bits (chain_ranges_fit), host floor kinds out of range or without floor1_y, a dense floor without dense_floor, decreasing host VQ offsets
// and, with pinned_only (a submit), host arrays that are not page-locked.  It writes nothing into the chain array and
// queues nothing.  The paths refuse a batch only on a CUDA error, and in one more case: the VQ entry's front-stage
// limits (channels, alignment, channels * n/2), which launch_prologue checks on the path that takes the batch.
static int walk_batch(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, bool pinned_only, BatchWalk *bw)
{
    int rc = check_batch_args(ctx, chains, n_chains, io);
    if (rc || n_chains == 0) return rc;
    BatchExtent &ext = bw->ext;
    bw->chains = chains;
    bw->walks.resize(n_chains);
    const bool planar = out_format_of(io->out_format).planar;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        ChainWalk &w = bw->walks[i] = walk_chain(c, [](uint32_t, const Geom &, bool, uint32_t, uint64_t, uint64_t) {});
        clip_to_window(c->stream, &w);
        if (!w.done) continue;
        if (planar && c->out_stride < w.written) return fail(ctx, LWB_ERR_BUFFER, "chain: out_stride smaller than the samples produced");
        if (!chain_ranges_fit(io, c, w)) return fail(ctx, LWB_ERR_BUFFER, "chain: a PCM, coefficient or packet-row range does not fit in 64 bits");
        ext.add(io, c, w);
        if (io->entry != LWB_ENTRY_SPECTRUM && (rc = scan_floor_kinds(ctx, io, c, w.done, &ext.need_dense, &ext.need_floor0))) return rc;
    }
    if (ext.need_dense && !io->dense_floor) return fail(ctx, LWB_ERR_INVALID, "dense_floor missing");
    if ((rc = check_vq_offsets(ctx, io, ext.r_lo, ext.r_hi))) return rc;
    if (!pinned_only || io->memory != LWB_MEM_HOST || ext.empty()) return LWB_OK;
    CU(ctx, cudaSetDevice(ctx->device));
    return check_page_locked(ctx, io, ext, chains[0].stream->setup->channels);
}

// Output windows (lwb_stream_set_window).  A clipped chain (ChainWalk::clipped) keeps the path its batch would take
// without a window: at end of stream nearly every step of a decode server has some stream ending, and routing those to
// the chain kernel would take most batches off k_long.  So it decodes its full output, laid out as the fused kernels
// want it -- planes of a multiple of g elements (8; 16 for i24, OutFormat::align), 16-byte aligned -- into scratch, and
// BatchArenas::download moves the samples it writes to their place with k_row_copy.  This writes bw->clip, the chain
// array the paths then decode: the clipped chains point into the scratch, the others are the caller's.  A host-memory
// batch's scratch follows the PCM extent in its staging (whose start moves down to a g-element boundary), so only
// written samples cross PCIe.  A device-memory batch's scratch is ctx->win, addressed from io->pcm by a wrapping element
// offset -- as the staged arenas are addressed from bases biased by their first element -- and placed at io->pcm's
// offset mod 16.  That offset is the byte distance over the element size modulo 2^64: the distance is a multiple of 16,
// so an exact quotient for 2- and 4-byte elements, and for 3-byte ones its product with the inverse of 3 mod 2^64.
static int place_clipped_chains(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, BatchWalk *bw)
{
    const OutFormat of = out_format_of(io->out_format);
    const uint64_t g = std::max(8u, of.align);
    auto region = [&](size_t i, uint64_t *stride) {
        const uint64_t K = chains[i].stream->setup->out_channels(), n = bw->walks[i].n_samples;
        *stride = (n + g - 1) & ~(g - 1);
        return of.planar ? K * *stride : (n * K + g - 1) & ~(g - 1);
    };
    uint64_t total = 0, stride;
    for (size_t i = 0; i < n_chains; i++)
        if (bw->walks[i].clipped()) total += region(i, &stride);
    if (!total) return LWB_OK;
    uint64_t at, end;
    if (io->memory == LWB_MEM_HOST) {
        BatchExtent &ext = bw->ext;
        at = (ext.o_hi + g - 1) & ~(g - 1);
        if (at < ext.o_hi || __builtin_add_overflow(at, total, &end) || __builtin_mul_overflow(end, (uint64_t)of.esz, &end))
            return fail(ctx, LWB_ERR_BUFFER, "chain: the staged PCM of a windowed batch does not fit in 64 bits");
        ext.o_lo &= ~(g - 1);
        ext.o_hi = at + total;
    } else {
        int rc;
        if ((rc = ensure(ctx, ctx->win, total * of.esz + 16))) return rc;
        const uintptr_t pcm = reinterpret_cast<uintptr_t>(io->pcm), win = reinterpret_cast<uintptr_t>(ctx->win.p) + (pcm & 15);
        const uint64_t d = (uint64_t)(win - pcm);
        at = of.esz == 3 ? d * 0xAAAAAAAAAAAAAAABull : d / of.esz;      // 3 * 0xAAAAAAAAAAAAAAAB == 1 mod 2^64
    }
    bw->clip.assign(chains, chains + n_chains);
    for (size_t i = 0; i < n_chains; i++) {
        if (!bw->walks[i].clipped()) continue;
        const uint64_t size = region(i, &stride);
        bw->clip[i].out_offset = at;
        bw->clip[i].out_stride = stride;
        at += size;
    }
    return LWB_OK;
}

// Walks one batch (walk_batch) and queues it on the first path that takes it.  Once the path has queued its work, the
// chain results and stream states of the walk are written; a refused batch changes neither.  A host-memory batch that
// queues work issues its ticket (BatchArenas::finish).
static int queue_batch(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, lwb_plan *prepared, bool pinned_only)
{
    if (!ctx || (!chains && n_chains) || !io) return LWB_ERR_INVALID;
    BatchWalk bw;
    int rc = walk_batch(ctx, chains, n_chains, io, pinned_only, &bw);
    if (rc || n_chains == 0) return rc;
    CU(ctx, cudaSetDevice(ctx->device));
    if ((rc = place_clipped_chains(ctx, chains, n_chains, io, &bw))) return rc;
    const lwb_chain *decode = bw.clip.empty() ? chains : bw.clip.data();
    if (prepared) prepared->captured = false; // the path that takes the batch captures it anew, if it can
    // An output mix is applied where one CTA holds every channel of a packet (k_chain) or by the four-kernel path: a batch
    // with a mixed chain skips the fused paths, as interleaved output does.
    size_t first = first_batch_path();
    for (size_t i = 0; i < n_chains && first < kChainPath; i++)
        if (chains[i].stream->setup->host.n_out) first = kChainPath;
    for (size_t k = first; k < std::size(kBatchPaths); k++) {
        bool handled = false;
        if ((rc = kBatchPaths[k](ctx, decode, n_chains, io, bw, &handled, prepared))) return rc;
        if (!handled) continue;
        if (prepared && !bw.clip.empty()) prepared->captured = false;   // a replay would not move the clipped samples
        for (size_t i = 0; i < n_chains; i++) set_chain_result(&chains[i], bw.walks[i]);
        commit_stream_states(chains, bw.walks);
        return LWB_OK;
    }
    return fail(ctx, LWB_ERR_INVALID, "internal: no batch path took the batch");
}

// One batch.  ticket == nullptr: the synchronous entry points, which return once a host-memory batch's PCM has landed
// (they wait for the ticket it issued).  Else lwb_submit_chains: *ticket identifies the batch's work, whatever its
// memory space, and nothing is waited for; a host-memory submit's arrays must be page-locked.
static int decode_chains_impl(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, lwb_plan *prepared,
                              uint64_t *ticket = nullptr)
{
    if (!ctx) return LWB_ERR_INVALID;
    const uint64_t issued = ctx->tickets_issued;
    int rc = queue_batch(ctx, chains, n_chains, io, prepared, ticket != nullptr);
    if (rc) return rc;
    if (!ticket) return ctx->tickets_issued != issued ? retire_tickets(ctx, ctx->tickets_issued, true) : LWB_OK;
    if (ctx->tickets_issued == issued) {        // a device-memory or empty batch (which may not have set the device)
        CU(ctx, cudaSetDevice(ctx->device));
        if ((rc = issue_ticket(ctx, nullptr))) return rc;
    }
    *ticket = ctx->tickets_issued;
    return LWB_OK;
}

extern "C" int lwb_decode_chains(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io)
{
    return decode_chains_impl(ctx, chains, n_chains, io, nullptr);
}

// ---------------------------------------------------------------------------------------------
// asynchronous batches
// ---------------------------------------------------------------------------------------------
extern "C" int lwb_submit_chains(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, uint64_t *ticket)
{
    if (!ctx || !ticket || (!chains && n_chains) || !io) return LWB_ERR_INVALID;
    return decode_chains_impl(ctx, chains, n_chains, io, nullptr, ticket);
}

extern "C" int lwb_ticket_query(lwb_ctx *ctx, uint64_t ticket, int *done)
{
    if (!ctx || !done || ticket == 0 || ticket > ctx->tickets_issued) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    const int rc = retire_tickets(ctx, ticket, false);
    *done = ticket <= ctx->tickets_done;
    return rc;
}

extern "C" int lwb_ticket_wait(lwb_ctx *ctx, uint64_t ticket)
{
    if (!ctx || ticket == 0 || ticket > ctx->tickets_issued) return LWB_ERR_INVALID;
    CU(ctx, cudaSetDevice(ctx->device));
    return retire_tickets(ctx, ticket, true);
}

// ---------------------------------------------------------------------------------------------
// many streams' states (lwb_streams_save / lwb_streams_load)
// ---------------------------------------------------------------------------------------------
// The state length slot `sl` moves: the stream's at call time for a save, the slot's for a load.
static uint32_t slot_len(const lwb_state_slot &sl, bool load)
{
    return load ? sl.len : (sl.stream->has ? sl.stream->plen : 0);
}

// Every refusal of a save or a load, before anything changes, and the element extent [*lo, *hi) of the slots' rows
// (empty: *hi <= *lo).  A slot's range must end inside the 64-bit address space in bytes, as chain_ranges_fit asks of a
// chain's ranges.
static int check_state_slots(lwb_ctx *ctx, const lwb_state_slot *slots, size_t n, int memory, const float *buf, const uint64_t *ticket,
                             bool load, uint64_t *lo, uint64_t *hi)
{
    if (!ctx) return LWB_ERR_INVALID;
    if ((!slots && n) || !buf || !ticket) return fail(ctx, LWB_ERR_INVALID, "streams_save / streams_load: a NULL argument");
    if (memory != LWB_MEM_HOST && memory != LWB_MEM_DEVICE) return fail(ctx, LWB_ERR_INVALID, "bad memory space");
    const uint64_t epoch = ++ctx->epoch;
    *lo = ~0ull;
    *hi = 0;
    for (size_t i = 0; i < n; i++) {
        const lwb_state_slot &sl = slots[i];
        lwb_stream *s = sl.stream;
        if (!s || s->ctx != ctx) return fail(ctx, LWB_ERR_INVALID, "slot: no stream, or a stream of another context");
        if (s->busy_epoch == epoch) return fail(ctx, LWB_ERR_INVALID, "a stream appears in two slots");
        s->busy_epoch = epoch;
        if (load && !sl.has && sl.len) return fail(ctx, LWB_ERR_INVALID, "slot: has == 0 with len != 0");
        if (load && sl.len > state_stride(s->setup)) return fail(ctx, LWB_ERR_BUFFER, "slot: len above blocksize_1 / 2 of the stream's setup");
        const uint64_t len = slot_len(sl, load);
        uint64_t end, bytes;
        if (__builtin_add_overflow(sl.offset, (uint64_t)s->setup->channels * len, &end) || __builtin_mul_overflow(end, (uint64_t)sizeof(float), &bytes))
            return fail(ctx, LWB_ERR_BUFFER, "slot: its range does not fit in 64 bits");
        if (!len) continue;
        *lo = std::min(*lo, sl.offset);
        *hi = std::max(*hi, end);
    }
    if (memory != LWB_MEM_HOST || *hi <= *lo) return LWB_OK;
    CU(ctx, cudaSetDevice(ctx->device));
    if (!page_locked(buf, *lo, *hi, sizeof(float)))
        return fail(ctx, LWB_ERR_INVALID, "host-memory streams_save / streams_load: buf is not page-locked (lwb_host_alloc, cudaHostAlloc or cudaHostRegister)");
    return LWB_OK;
}

// Queues one k_row_copy launch over the (slot, channel) rows of nonzero length: stream state row c <-> dev + offset - base
// + c * len.  Its descriptors go through the staging ring like a batch's.
static int queue_state_rows(lwb_ctx *ctx, const lwb_state_slot *slots, size_t n, float *dev, uint64_t base, bool load)
{
    size_t rows = 0;
    for (size_t i = 0; i < n; i++)
        if (slot_len(slots[i], load)) rows += slots[i].stream->setup->channels;
    if (!rows) return LWB_OK;
    Staging *st;
    int rc;
    if ((rc = acquire_staging(ctx, rows * sizeof(RowCopy), &st)) || (rc = ensure(ctx, ctx->state_rows, rows * sizeof(RowCopy)))) return rc;
    RowCopy *h = (RowCopy *)st->h;
    size_t k = 0;
    for (size_t i = 0; i < n; i++) {
        const lwb_stream *s = slots[i].stream;
        const uint32_t len = slot_len(slots[i], load);
        for (unsigned c = 0; len && c < s->setup->channels; c++) {
            float *row = s->d_state + (size_t)c * state_stride(s->setup), *b = dev + (slots[i].offset - base) + (uint64_t)c * len;
            h[k++] = load ? RowCopy{b, row, len * sizeof(float)} : RowCopy{row, b, len * sizeof(float)};
        }
    }
    if ((rc = upload_staging(ctx, st, h, ctx->state_rows.p, rows * sizeof(RowCopy), ctx->stream))) return rc;
    return run_steps(ctx, StepArgs(), std::vector<Step>(1, Step{LWB_KERNEL_ROW_COPY, ctx->state_rows.p, rows, nullptr}));
}

// A save (load == false) or a load, queued on the compute stream with its ticket.  Host memory is staged in the next host
// arena set, which the set's previous user releases on the GPU (ArenaSet::done) and this call's ticket releases in turn.
// slots_w: the save's slots, written once the work is queued (nullptr for a load).
static int move_states(lwb_ctx *ctx, bool load, lwb_state_slot *slots_w, const lwb_state_slot *slots, size_t n, int memory, float *buf,
                       uint64_t *ticket)
{
    uint64_t lo, hi;
    int rc = check_state_slots(ctx, slots, n, memory, buf, ticket, load, &lo, &hi);
    if (rc) return rc;
    CU(ctx, cudaSetDevice(ctx->device));
    ArenaSet *set = nullptr;
    if (memory == LWB_MEM_DEVICE || hi <= lo) {
        if ((rc = queue_state_rows(ctx, slots, n, buf, 0, load))) return rc;
    } else {
        set = &ctx->host_sets[ctx->host_next];
        ctx->host_next = (ctx->host_next + 1) % kHostSets;
        const size_t bytes = (size_t)(hi - lo) * sizeof(float);
        if ((rc = ensure(ctx, set->coeffs, bytes, set->done))) return rc;
        CU(ctx, cudaStreamWaitEvent(ctx->stream, set->done, 0));
        float *stage = (float *)set->coeffs.p;
        if (load) CU(ctx, cudaMemcpyAsync(stage, buf + lo, bytes, cudaMemcpyHostToDevice, ctx->stream));
        rc = queue_state_rows(ctx, slots, n, stage, lo, load);
        if (!rc && !load) {       // exactly the slots' rows go home: the gaps between them are the caller's
            std::vector<PcmSpan> spans;
            std::vector<PcmCopy> copies;
            for (size_t i = 0; i < n; i++)
                if (const uint32_t len = slot_len(slots[i], false)) spans.push_back(PcmSpan{slots[i].offset, (uint64_t)slots[i].stream->setup->channels * len});
            plan_pcm_copies(spans, (uint64_t)INT32_MAX / sizeof(float), copies);
            for (const PcmCopy &cp : copies) {
                float *dst = buf + cp.off;
                const float *src = stage + (cp.off - lo);
                cudaError_t e = cp.height == 1 ? cudaMemcpyAsync(dst, src, cp.width * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream)
                                               : cudaMemcpy2DAsync(dst, cp.pitch * sizeof(float), src, cp.pitch * sizeof(float), cp.width * sizeof(float),
                                                                   cp.height, cudaMemcpyDeviceToHost, ctx->stream);
                if (e != cudaSuccess) {
                    rc = fail(ctx, LWB_ERR_CUDA, "streams_save: copy to host", e);
                    break;
                }
            }
        }
        if (rc) {               // the set's next user still waits behind whatever this call queued
            cudaEventRecord(set->done, ctx->stream);
            cudaGetLastError();
            return rc;
        }
    }
    if ((rc = issue_ticket(ctx, set))) return rc;
    *ticket = ctx->tickets_issued;
    for (size_t i = 0; i < n; i++) {
        lwb_stream *s = slots[i].stream;
        if (load) {
            s->has = slots[i].has != 0;
            s->plen = slots[i].len;
        } else {
            slots_w[i].len = slot_len(slots[i], false);
            slots_w[i].has = s->has ? 1 : 0;
        }
    }
    if (load) ctx->state_gen++;     // contents changed even where the shape did not: prepared batches plan again
    return LWB_OK;
}

extern "C" int lwb_streams_save(lwb_ctx *ctx, lwb_state_slot *slots, size_t n, int memory, float *buf, uint64_t *ticket)
{
    return move_states(ctx, false, slots, slots, n, memory, buf, ticket);
}

extern "C" int lwb_streams_load(lwb_ctx *ctx, const lwb_state_slot *slots, size_t n, int memory, const float *buf, uint64_t *ticket)
{
    // (a load only reads buf: move_states writes through it on a save alone)
    return move_states(ctx, true, nullptr, slots, n, memory, const_cast<float *>(buf), ticket);
}

// ---------------------------------------------------------------------------------------------
// what the stream batcher (batcher.h) needs of setups and streams
// ---------------------------------------------------------------------------------------------
namespace lwfb {
SetupShape setup_shape(const lwb_setup *su) { return SetupShape{su->ctx, su->channels, su->bs0, su->bs1}; }

const lwb_setup *stream_setup(const lwb_stream *s) { return s->setup; }

StreamFlags stream_flags(const lwb_stream *s) { return StreamFlags{s->has, s->plen}; }

void set_stream_flags(lwb_stream *s, StreamFlags f) { set_stream_state(s, f.has, f.plen); }

// The walk lwb_submit_chains makes of this batch (walk_batch), queuing nothing.
int check_submit(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io)
{
    BatchWalk bw;
    return walk_batch(ctx, chains, n_chains, io, true, &bw);
}
}  // namespace lwfb

// ---------------------------------------------------------------------------------------------
// prepared batches
// ---------------------------------------------------------------------------------------------
extern "C" int lwb_plan_create(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, lwb_plan **out)
{
    if (!ctx || !out || (!chains && n_chains) || !io) return LWB_ERR_INVALID;
    lwb_plan *p = new (std::nothrow) lwb_plan();
    if (!p) return LWB_ERR_BUFFER;
    p->ctx = ctx;
    p->chains = chains;
    p->n_chains = n_chains;
    p->io = *io;
    *out = p;
    return LWB_OK;
}

extern "C" void lwb_plan_destroy(lwb_plan *p)
{
    if (!p) return;
    if (p->desc.p || p->pro.p) {
        cudaSetDevice(p->ctx->device);
        cudaStreamSynchronize(p->ctx->stream);
        if (p->desc.p) cudaFree(p->desc.p);
        if (p->pro.p) cudaFree(p->pro.p);
    }
    delete p;
}

// Whether a stream of the plan has an output window that may clip it: its counters move at every execution, which a
// replay would not do.
static bool plan_has_window(const lwb_plan *p)
{
    for (size_t i = 0; i < p->n_chains; i++)
        if (p->chains[i].stream->skip_left || p->chains[i].stream->limit_left != ~0ull) return true;
    return false;
}

extern "C" int lwb_plan_execute(lwb_plan *p)
{
    if (!p) return LWB_ERR_INVALID;
    lwb_ctx *ctx = p->ctx;
    if (!p->captured || p->gen != ctx->state_gen || first_batch_path() != 0 || (ctx->windows_set && plan_has_window(p)))
        return decode_chains_impl(ctx, p->chains, p->n_chains, &p->io, p);
    // steady state: nothing about the batch or the stream states has changed shape since the descriptors were
    // built -- the per-chain results in the caller's array and the stream states are still right: just launch.
    // (Host floor arrays change from step to step and are uploaded again; device floor arrays are read in place.)
    CU(ctx, cudaSetDevice(ctx->device));
    int rc;
    if (p->front.n && (rc = front_stages_run(ctx, &p->io, p->front))) return rc;    // they write ctx->spec, which the steps read
    return run_steps(ctx, p->args, p->steps);
}

// ---------------------------------------------------------------------------------------------
// one packet
// ---------------------------------------------------------------------------------------------
static int one_packet(lwb_stream *s, int entry, uint8_t mode, int prev_flag, int next_flag, const float *coeffs,
                      const lwb_packet *pkt, int out_format, void *out, size_t cap, size_t *n_samples)
{
    if (!s || !coeffs || !out || !n_samples) return LWB_ERR_INVALID;
    *n_samples = 0;
    Geom g;
    int rc = geometry(s->setup, mode, prev_flag, next_flag, &g);
    if (rc) return rc;
    const size_t produce = s->has ? g.rs - g.ls : 0;
    if (produce > cap) return LWB_ERR_BUFFER;          // checked before anything is consumed
    uint8_t m = mode, pf = (uint8_t)(prev_flag != 0), nf = (uint8_t)(next_flag != 0);
    lwb_chain c;
    std::memset(&c, 0, sizeof(c));
    c.stream = s;
    c.n_packets = 1;
    c.mode_numbers = &m;
    c.prev_window_flags = &pf;
    c.next_window_flags = &nf;
    c.out_stride = cap;
    lwb_batch_io io;
    std::memset(&io, 0, sizeof(io));
    io.entry = entry;
    io.memory = LWB_MEM_HOST;
    io.coeffs = coeffs;
    if (pkt) {
        io.dense_floor = pkt->dense_floor;
        io.floor_kind = pkt->floor_kind;
        io.floor1_y = pkt->floor1_y;
    }
    io.out_format = out_format;
    io.pcm = out;
    rc = lwb_decode_chains(s->ctx, &c, 1, &io);
    if (rc) return rc;
    if (c.status) return c.status;
    *n_samples = c.n_samples;
    return LWB_OK;
}

extern "C" int lwb_decode_packet(lwb_stream *s, const lwb_packet *pkt, int out_format, void *out, size_t cap,
                                 size_t *n_samples)
{
    if (!pkt || !pkt->floor_kind || !pkt->residue) return LWB_ERR_INVALID;
    return one_packet(s, LWB_ENTRY_RESIDUE, pkt->mode_number, pkt->prev_window_flag, pkt->next_window_flag,
                      pkt->residue, pkt, out_format, out, cap, n_samples);
}

extern "C" int lwb_decode_spectrum(lwb_stream *s, uint8_t mode, int prev_flag, int next_flag, const float *spectrum,
                                   int out_format, void *out, size_t cap, size_t *n_samples)
{
    return one_packet(s, LWB_ENTRY_SPECTRUM, mode, prev_flag, next_flag, spectrum, nullptr, out_format, out, cap,
                      n_samples);
}

// ---------------------------------------------------------------------------------------------
// debug taps (lib.rs:56-94): intermediates of one packet, state untouched
// ---------------------------------------------------------------------------------------------
extern "C" int lwb_debug_packet_taps(lwb_stream *s, const lwb_packet *pkt, float *post_inverse, float *pre_mdct,
                                     float *post_mdct)
{
    if (!s || !pkt || !pkt->floor_kind || !pkt->residue) return LWB_ERR_INVALID;
    lwb_ctx *ctx = s->ctx;
    const lwb_setup *su = s->setup;
    Geom g;
    int rc = geometry(su, pkt->mode_number, pkt->prev_window_flag, pkt->next_window_flag, &g);
    if (rc) return rc;
    CU(ctx, cudaSetDevice(ctx->device));
    const size_t C = su->channels, n2 = g.n >> 1;
    bool need_dense = false, need_y = false, need_floor0 = false;
    for (size_t c = 0; c < C; c++) {
        const uint8_t kd = pkt->floor_kind[c];
        if (kd > LWB_FLOOR_ZERO) return LWB_ERR_INVALID;
        if (kd == LWB_FLOOR_ZERO && !su->floor0_described(su->mappings[g.mapping].floor_of_channel[c])) return LWB_ERR_INVALID;
        need_dense |= kd == LWB_FLOOR_DENSE;
        need_y |= kd == LWB_FLOOR_ONE || kd == LWB_FLOOR_ZERO;
        need_floor0 |= kd == LWB_FLOOR_ZERO;
    }
    if ((need_dense && !pkt->dense_floor) || (need_y && !pkt->floor1_y)) return LWB_ERR_INVALID;
    Staging *slot;
    if ((need_floor0 && (rc = ensure(ctx, ctx->floor0, C * n2 * 4))) ||
        (rc = ensure(ctx, ctx->ordered.coeffs, C * n2 * 4)) || (rc = ensure(ctx, ctx->spec, C * n2 * 4)) ||
        (rc = ensure(ctx, ctx->x, C * g.n * 4)) || (rc = ensure(ctx, ctx->ordered.kinds, C)) ||
        (rc = ensure(ctx, ctx->ordered.ys, C * LWB_MAX_POSTS * 4)) || (rc = ensure(ctx, ctx->ordered.dense, C * n2 * 4)) ||
        (rc = ensure(ctx, ctx->desc, sizeof(DevPacket))) || (rc = acquire_staging(ctx, sizeof(DevPacket), &slot)))
        return rc;
    DevPacket *d = (DevPacket *)slot->h;
    std::memset(d, 0, sizeof(*d));
    d->setup = su->d_setup;
    d->state = s->d_state;
    d->prev_packet = -1;
    d->state_stride = (uint32_t)state_stride(su);
    d->n = (uint16_t)g.n;
    d->ls = (uint16_t)g.ls; d->rs = (uint16_t)g.rs; d->re = (uint16_t)g.re;
    d->blockflag = g.blockflag; d->mapping = g.mapping; d->slope_sel = g.slope_sel;
    d->channels = (uint8_t)C;
    cudaStream_t st = ctx->stream;
    if ((rc = upload_staging(ctx, slot, d, ctx->desc.p, sizeof(*d), st))) return rc;
    CU(ctx, cudaMemcpyAsync(ctx->ordered.coeffs.p, pkt->residue, C * n2 * 4, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(ctx->ordered.kinds.p, pkt->floor_kind, C, cudaMemcpyHostToDevice, st));
    if (need_y) CU(ctx, cudaMemcpyAsync(ctx->ordered.ys.p, pkt->floor1_y, C * LWB_MAX_POSTS * 4, cudaMemcpyHostToDevice, st));
    if (need_dense) CU(ctx, cudaMemcpyAsync(ctx->ordered.dense.p, pkt->dense_floor, C * n2 * 4, cudaMemcpyHostToDevice, st));
    const DevPacket *dp = (const DevPacket *)ctx->desc.p;
    if (post_inverse) {
        // audio.rs:1004 tap: coupling only.  The prologue runs with every channel's floor a dense unit curve, so that
        // floor x residue leaves the decoupled residue unchanged.  Curve and kinds sit in the IMDCT scratch ctx->x
        // (C * n floats), which the tap uses again only after this prologue.
        float *unit = (float *)ctx->x.p;
        uint8_t *unit_kinds = (uint8_t *)(unit + C * n2);
        const std::vector<float> ones(C * n2, 1.0f);
        CU(ctx, cudaMemcpyAsync(unit, ones.data(), C * n2 * 4, cudaMemcpyHostToDevice, st));
        CU(ctx, cudaMemsetAsync(unit_kinds, LWB_FLOOR_DENSE, C, st));
        if ((rc = launch(ctx, LWB_KERNEL_PROLOGUE, k_prologue, dim3(1), dim3(kPrologueThreads), prologue_smem(su->channels, su->bs1), dp,
                         (const float *)ctx->ordered.coeffs.p, (const float *)unit, (const uint8_t *)unit_kinds,
                         (const uint32_t *)ctx->ordered.ys.p, (float *)ctx->spec.p, (const float *)nullptr)))
            return rc;
        CU(ctx, cudaMemcpyAsync(post_inverse, ctx->spec.p, C * n2 * 4, cudaMemcpyDeviceToHost, st));
    }
    float *zero = need_floor0 ? (float *)ctx->floor0.p : nullptr;
    if (zero && (rc = launch_floor0_curves(ctx, dp, 1, (unsigned)C, (const uint8_t *)ctx->ordered.kinds.p, (const uint32_t *)ctx->ordered.ys.p, zero)))
        return rc;
    if ((rc = launch(ctx, LWB_KERNEL_PROLOGUE, k_prologue, dim3(1), dim3(kPrologueThreads), prologue_smem(su->channels, su->bs1), dp, (const float *)ctx->ordered.coeffs.p,
                     (const float *)ctx->ordered.dense.p, (const uint8_t *)ctx->ordered.kinds.p, (const uint32_t *)ctx->ordered.ys.p,
                     (float *)ctx->spec.p, (const float *)zero)))
        return rc;
    if (pre_mdct) CU(ctx, cudaMemcpyAsync(pre_mdct, ctx->spec.p, C * n2 * 4, cudaMemcpyDeviceToHost, st));
    if (post_mdct) {
        if ((rc = launch(ctx, LWB_KERNEL_IMDCT, k_imdct, dim3(1, (unsigned)C), dim3(kImdctThreads), g.n * sizeof(float), dp,
                         (const float *)ctx->spec.p, (float *)ctx->x.p)))
            return rc;
        CU(ctx, cudaMemcpyAsync(post_mdct, ctx->x.p, C * g.n * 4, cudaMemcpyDeviceToHost, st));
    }
    CU(ctx, cudaStreamSynchronize(st));
    return LWB_OK;
}

