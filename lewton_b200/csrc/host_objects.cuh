// host_objects.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the opaque objects behind the handles (ctx, setup, stream, plan), error / buffer helpers and the
// window geometry of audio.rs:1056-1073.
#pragma once

// ---------------------------------------------------------------------------------------------
// objects
// ---------------------------------------------------------------------------------------------
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

// pinned staging for one batch's descriptors; `ev` marks the end of the copy that reads it
struct Staging {
    void *h = nullptr;
    size_t cap = 0;
    cudaEvent_t ev = nullptr;
    bool pending = false;
};

// CachedBlocksizeDerived (header_cached.rs:27-31) on the device, shared by all setups of a context with the same tables
struct CachedTables {
    DevTables dt;                  // device pointers; dt.pack = the fused kernels' twiddle pack (bs 11: k_long, bs 8: k_short)
    std::vector<float> a, b, c, w; // host copies: the cache key
    std::vector<uint32_t> br;
    std::vector<void *> allocs;
};

struct lwb_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_in = nullptr, copy_out = nullptr;
    cudaEvent_t ev_in[64] = {}, ev_done[65] = {};      // per chunk of a host-memory batch; [64] orders the copy streams
    // fused path: descriptor arrays are double buffered and uploaded on the copy stream so that the
    // upload of step k+1 overlaps kernel k; tickets come from a pool zeroed once per wrap
    DevBuf runs_buf[2];
    cudaEvent_t ev_desc[2] = {}, ev_kdone[2] = {};
    int runs_par = 0;
    uint32_t ticket_next = 0;
    uint64_t epoch = 0;            // batch counter: lwb_stream::busy_epoch == epoch <=> the stream already sits in this batch
    uint64_t state_gen = 1;        // bumped whenever any stream's (has, len) changes: plans key on it
    std::string err;
    uint64_t launches = 0;
    uint64_t kernel_launches[LWB_KERNEL_COUNT] = {};   // per LWB_KERNEL_* id; they sum to `launches`
    std::vector<PcmSpan> pcm_spans;        // scratch of copy_pcm_to_host
    std::vector<PcmCopy> pcm_copies;
    std::deque<CachedTables> tables;       // (deque: setups hold copies of dt, growth never moves an entry)
    // grow-only device arenas
    DevBuf coeffs, dense, pcm, spec, segtab, vqoff, vqrec, magic, x, desc, kinds, ys, chains, ticket, cdesc, cbytes;
    Staging stage[3];              // ring: a batch's descriptors are written while the previous copies may still run
    int stage_next = 0;
    // pinned staging for descriptors (four-kernel path)
    void *h_desc = nullptr;
    size_t h_desc_cap = 0;
    size_t x_cap_elems = (size_t)64 << 20;     // IMDCT scratch per round of the generic path (256 MiB)
};

struct lwb_setup {
    lwb_ctx *ctx = nullptr;
    DevSetup host;                 // device pointers inside
    DevSetup *d_setup = nullptr;
    std::vector<void *> allocs;
    uint8_t channels = 0, bs0 = 0, bs1 = 0;
    uint32_t n_modes = 0;
    uint32_t n_mappings = 0;
    std::vector<DevMapping> mappings;   // host copy (validation)
};

struct MixRound { size_t r0, nr, s0, ns, c0, nc, x0, nx, g0, ng, flat, nm; };   // LongRun / ShortRun / ChainDesc / RowCopy / burst-group ranges of one
                                                                            // round; flat: the one-pass round (static deal, k_long_s);
                                                                            // nm: groups of k_mid (path_mid.cuh, from the buffer's start)
struct RowCopy { const float *src; float *dst; uint32_t n4, pad; };  // n4 float4s, copied in front of the round's kernels
struct MixLaunch {
    char *db; size_t off_sr, off_cd, off_by, off_rc, off_sg;
    const float *pack, *spack, *w_short, *mpack; int ls, mid_kb; bool i16, residue; int out_format; unsigned warps; size_t smem; int n1max, wpc, np;
    const float *coeffs, *dense; const uint8_t *kinds; const uint32_t *ys; void *pcm;
};

// One launch of the residue entry's front stages (k_floor1_segments + k_prologue_fused, or k_prologue): floor x
// decoupled residue -> ctx->spec for a list of packets with one channel count.  The packet list holds absolute element
// offsets and packet rows; the arenas are biased instead (the spectrum by c_lo, floor / VQ arrays by their staging).
struct FrontStages {
    const DevPacket *pk = nullptr;     // device packet list
    size_t n = 0;
    unsigned C = 0;
    bool fast = false;                 // the two-kernel form; else k_prologue with smem_old bytes of shared memory
    size_t smem_old = 0;
    int n2max = 0;                     // largest n/2 among the packets
    uint64_t c_lo = 0;                 // element offset of ctx->spec[0]
    uint64_t r_lo = 0, r_hi = 0;       // packet rows of the floor / VQ arrays
    bool dense = false;                // whether the dense floor arena is passed
};

struct lwb_plan {
    lwb_ctx *ctx = nullptr;
    lwb_chain *chains = nullptr;
    size_t n_chains = 0;
    lwb_batch_io io;
    // captured launch sequence (valid while ctx->state_gen == gen): the front stages if front.n, then either the
    // rounds of mix_launch or, when there are none, one k_long over `runs`.  Every path that captures a residue-entry
    // batch sets `front`; a spectrum-entry plan never does.
    bool captured = false;
    uint64_t gen = 0;
    FrontStages front;
    DevBuf runs, pro, mix;             // descriptors the capture owns: k_long runs, the long path's front stages, the rest
    uint32_t n_groups = 0;
    const float *pack = nullptr;
    bool i16 = false;
    MixLaunch mix_launch;
    std::vector<MixRound> mix_rounds;
};

struct lwb_stream {
    lwb_ctx *ctx = nullptr;
    const lwb_setup *setup = nullptr;
    float *d_state = nullptr;      // [channels][n1/2]
    bool has = false;              // PreviousWindowRight.data.is_some()
    uint32_t plen = 0;             // per-channel length of the saved right half
    uint64_t busy_epoch = 0;       // guards against one stream appearing twice in a batch
};

static inline void set_stream_state(lwb_stream *s, bool has, uint32_t plen)
{
    if (s->has != has || s->plen != plen) {
        s->has = has;
        s->plen = plen;
        s->ctx->state_gen++;
    }
}

static int fail(lwb_ctx *ctx, int code, const char *what, cudaError_t e = cudaSuccess)
{
    if (ctx) {
        ctx->err = what;
        if (e != cudaSuccess) {
            ctx->err += ": ";
            ctx->err += cudaGetErrorString(e);
        }
    }
    return code;
}

// One kernel launch enqueued: the total and the count of its kernel.  Only launch() and launched() (path_generic.cuh)
// call this; tests/test_cabi_cpu.py checks that every launch site goes through one of them.
static inline void count_launch(lwb_ctx *ctx, int kernel_id)
{
    ctx->launches++;
    ctx->kernel_launches[kernel_id]++;
}

#define CU(ctx, call)                                                        \
    do {                                                                     \
        cudaError_t e__ = (call);                                            \
        if (e__ != cudaSuccess) return fail((ctx), LWB_ERR_CUDA, #call, e__); \
    } while (0)

static int ensure(lwb_ctx *ctx, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return LWB_OK;
    if (b.p) {
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        CU(ctx, cudaFree(b.p));
        b.p = nullptr;
        b.cap = 0;
    }
    size_t want = bytes + bytes / 8 + 4096;
    CU(ctx, cudaMalloc(&b.p, want));
    b.cap = want;
    ctx->state_gen++;              // captured plans may hold pointers into the arena that just moved
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// host-memory pipeline and fused-kernel tickets
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kTicketPool = 1024;

// The per-context events of the host-memory pipeline and the fused kernels' ticket pool, made once by lwb_ctx_create.
static int create_pipeline_objects(lwb_ctx *ctx)
{
    for (int k = 0; k < 65; k++) {
        if (k < 64) CU(ctx, cudaEventCreateWithFlags(&ctx->ev_in[k], cudaEventDisableTiming));
        CU(ctx, cudaEventCreateWithFlags(&ctx->ev_done[k], cudaEventDisableTiming));
    }
    for (int k = 0; k < 2; k++) {
        CU(ctx, cudaEventCreateWithFlags(&ctx->ev_desc[k], cudaEventDisableTiming));
        CU(ctx, cudaEventCreateWithFlags(&ctx->ev_kdone[k], cudaEventDisableTiming));
    }
    return ensure(ctx, ctx->ticket, kTicketPool * sizeof(unsigned int));
}

// The ticket of one k_long launch; the pool is zeroed on the compute stream once per wrap.
static int next_ticket(lwb_ctx *ctx, unsigned int **ticket)
{
    if (ctx->ticket_next % kTicketPool == 0)
        CU(ctx, cudaMemsetAsync(ctx->ticket.p, 0, kTicketPool * sizeof(unsigned int), ctx->stream));
    *ticket = (unsigned int *)ctx->ticket.p + (ctx->ticket_next++ % kTicketPool);
    return LWB_OK;
}

// The copy streams must not run ahead of work already queued on the compute stream that still reads or writes the
// arenas (a previous call, a descriptor upload): order them behind it.
static int order_copies_behind_compute(lwb_ctx *ctx)
{
    CU(ctx, cudaEventRecord(ctx->ev_done[64], ctx->stream));
    CU(ctx, cudaStreamWaitEvent(ctx->copy_in, ctx->ev_done[64], 0));
    CU(ctx, cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[64], 0));
    return LWB_OK;
}

// Chunks of a host-memory batch, whose H2D / kernels / D2H overlap on three streams: one per 32 MiB of input, at most
// 8 and at most one per chain.  LWB_E2E_CHUNKS=n sets the count, up to what ev_in / ev_done can index.
static size_t host_chunks(size_t in_bytes, size_t n_chains)
{
    if (const char *e = getenv("LWB_E2E_CHUNKS")) return std::max<size_t>(1, std::min<size_t>((size_t)atol(e), std::min<size_t>(64, n_chains)));
    return std::min<size_t>(std::max<size_t>(1, in_bytes >> 25), std::min<size_t>(8, n_chains));
}

static size_t elem_size(int fmt) { return (fmt == LWB_OUT_F32_PLANAR || fmt == LWB_OUT_F32_INTERLEAVED) ? 4 : 2; }
static bool is_planar(int fmt) { return fmt == LWB_OUT_F32_PLANAR || fmt == LWB_OUT_I16_PLANAR; }

// D2H of the PCM that chains [i0, i1) produced, from the staging buffer `stage`, which holds arena element `obase` at
// its start.  Only the write set is copied (pcm_copy_plan.h): the gaps between planes and between chains are the
// caller's memory, and the kernels never wrote them in the staging buffer.
static int copy_pcm_to_host(lwb_ctx *ctx, const lwb_batch_io *io, const lwb_chain *chains, size_t i0, size_t i1,
                            const void *stage, uint64_t obase, cudaStream_t st)
{
    const size_t esz = elem_size(io->out_format);
    const bool planar = is_planar(io->out_format);
    ctx->pcm_spans.clear();
    for (size_t i = i0; i < i1; i++) {
        const lwb_chain *c = &chains[i];
        pcm_chain_spans(planar, c->stream->setup->channels, c->out_offset, c->out_stride, c->n_samples, ctx->pcm_spans);
    }
    plan_pcm_copies(ctx->pcm_spans, (uint64_t)INT32_MAX / esz, ctx->pcm_copies);
    for (const PcmCopy &cp : ctx->pcm_copies) {
        char *dst = (char *)io->pcm + cp.off * esz;
        const char *src = (const char *)stage + (cp.off - obase) * esz;
        if (cp.height == 1) CU(ctx, cudaMemcpyAsync(dst, src, cp.width * esz, cudaMemcpyDeviceToHost, st));
        else CU(ctx, cudaMemcpy2DAsync(dst, cp.pitch * esz, src, cp.pitch * esz, cp.width * esz, cp.height, cudaMemcpyDeviceToHost, st));
    }
    return LWB_OK;
}

// The fused kernels load coefficients with TMA bulk copies and store PCM with vector stores, which need 16-byte aligned
// addresses.  Element offsets that are multiples of 4 keep that when the arenas are 16-byte aligned: the library's
// staging of host-memory batches always is, a caller's device arena may not be (the chain kernel takes those).
static bool device_arenas_aligned(const lwb_batch_io *io)
{
    if (io->memory != LWB_MEM_DEVICE) return true;
    return ((reinterpret_cast<uintptr_t>(io->coeffs) | reinterpret_cast<uintptr_t>(io->pcm) |
             reinterpret_cast<uintptr_t>(io->dense_floor)) & 15) == 0;
}

static int ensure_pinned(lwb_ctx *ctx, size_t bytes)
{
    if (bytes <= ctx->h_desc_cap) return LWB_OK;
    if (ctx->h_desc) {
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        cudaFreeHost(ctx->h_desc);
        ctx->h_desc = nullptr;
        ctx->h_desc_cap = 0;
    }
    size_t want = bytes * 2 + 4096;
    CU(ctx, cudaHostAlloc(&ctx->h_desc, want, cudaHostAllocDefault));
    ctx->h_desc_cap = want;
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// window geometry, audio.rs:1056-1073 (and its twin :889-908)
// ---------------------------------------------------------------------------------------------
struct Geom {
    uint32_t n, ls, le, rs, re;
    uint8_t blockflag, slope_sel, mapping;
};

static int geometry(const lwb_setup *su, uint8_t mode, int prev_flag, int next_flag, Geom *g)
{
    if (mode >= su->n_modes) return LWB_ERR_BAD_FORMAT;          // audio.rs:926-930
    const bool lng = su->host.mode_blockflag[mode] != 0;
    const uint32_t n = 1u << (lng ? su->bs1 : su->bs0);
    const uint32_t n0 = 1u << su->bs0;
    const bool prev = lng ? (prev_flag != 0) : true;             // short blocks: map_or(true, ..)
    const bool next = lng ? (next_flag != 0) : true;
    g->n = n;
    g->blockflag = lng;
    g->mapping = su->host.mode_mapping[mode];
    if (prev) { g->ls = 0; g->le = n >> 1; g->slope_sel = lng; }
    else { g->ls = (n - n0) >> 2; g->le = (n + n0) >> 2; g->slope_sel = 0; }
    if (next) { g->rs = n >> 1; g->re = n; }
    else { g->rs = (n * 3 - n0) >> 2; g->re = (n * 3 + n0) >> 2; }
    return LWB_OK;
}

