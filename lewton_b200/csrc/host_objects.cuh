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

// pinned staging for one batch's descriptors (the four-kernel path: one round's); `ev` marks the end of the copy that reads it
struct Staging {
    void *h = nullptr;
    size_t cap = 0;
    cudaEvent_t ev = nullptr;
    bool pending = false;
};

// Device copies of one batch's host arrays (coefficients, dense floors, floor and VQ arrays) and its PCM before the
// D2H.  Host-memory batches take the context's kHostSets sets in turn, so that the uploads of one batch overlap the
// kernels and copies of the one before it: a set is reused only behind `done`, which is recorded after the last kernel
// and the last D2H of the batch that used it last.
struct ArenaSet {
    DevBuf coeffs, dense, pcm, kinds, ys, vqoff, vqrec;
    cudaEvent_t done = nullptr;
};
constexpr int kHostSets = 2;

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
    bool windows_set = false;      // lwb_stream_set_window has been called on a stream of this ctx
    std::string err;
    uint64_t launches = 0;
    uint64_t kernel_launches[LWB_KERNEL_COUNT] = {};   // per LWB_KERNEL_* id; they sum to `launches`
    std::vector<PcmSpan> pcm_spans;        // scratch of copy_pcm_to_host
    std::vector<PcmCopy> pcm_copies;
    std::deque<CachedTables> tables;       // (deque: setups hold copies of dt, growth never moves an entry)
    // grow-only device arenas
    DevBuf spec, segtab, magic, x, desc, chains, ticket, cdesc, cbytes;
    DevBuf floor0;                 // floor-0 curves of LWB_FLOOR_ZERO rows (k_floor0_curves), laid out like spec
    DevBuf state_rows;             // RowCopy descriptors, in compute-stream order: lwb_streams_save / load, clipped chains
    DevBuf win;                    // device-memory batches: the full output of their clipped chains (BatchWalk::clip)
    ArenaSet host_sets[kHostSets]; // host-memory batches, in turn
    int host_next = 0;
    ArenaSet ordered;              // in compute-stream order: device-memory batches' host floor arrays, the debug taps
    Staging stage[3];              // ring: a batch's descriptors are written while the previous copies may still run
    int stage_next = 0;
    std::vector<void *> stage_old; // staging outgrown, freed with the context (cudaFreeHost waits for the whole device)
    // completion tickets (lwb_submit_chains, and every host-memory batch): ticket t's event is ticket_events[t -
    // tickets_done - 1]; they are retired in order
    uint64_t tickets_issued = 0, tickets_done = 0;
    std::deque<cudaEvent_t> ticket_events;
    std::vector<cudaEvent_t> spare_events;
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
    std::vector<uint8_t> floor_types;   // LWB_FLOOR_TYPE_* per floor
    std::vector<DevFloor0> floor0;      // host copy of host.floor0 (empty: no floor-0 description)
    mutable bool streams_opened = false; // lwb_setup_set_floor0 and lwb_setup_set_output_mix are refused from then on
    bool floor0_described(uint32_t fi) const { return fi < floor0.size() && floor0[fi].order != 0; }
    // K: the channels a chain of this setup writes (lwb_setup_set_output_mix)
    unsigned out_channels() const { return host.n_out ? host.n_out : channels; }
};

// One row for k_row_copy: `bytes` from src to dst at any byte alignment (rows of any sample type, 3-byte ones included)
struct RowCopy { const void *src; void *dst; uint64_t bytes; };
constexpr int kRowCopyThreads = 256;
struct ChainShape { unsigned warps; size_t smem; int n1max, wpc, np; };     // k_chain's block and shared memory

// One launch of a batch path (run_steps, path_generic.cuh): the kernel's LWB_KERNEL_* id, a device pointer to its
// descriptors -- runs or run groups (LongRun, ShortRun), ChainDescs or RowCopys -- their count (groups for k_long, k_mid
// and k_short_g) and the twiddle pack it uses.
struct Step {
    int kernel;
    const void *desc;
    size_t n;
    const float *pack;
};

// What the steps of one batch share.  Set member by member; what a path does not launch stays zero.
struct StepArgs {
    void *pcm = nullptr;                                    // PCM arena (k_chain; the runs carry their own pointers)
    int out_format = LWB_OUT_F32_PLANAR;
    const float *w_short = nullptr;                         // k_long / k_long_s: short window and ls of transitional blocks
    int ls = 0;
    int mid_kb = 0;                                         // k_mid: 1 for n = 1024, 2 for n = 512
    ChainShape chain = {};                                  // k_chain
    const uint8_t *bytes = nullptr;                         // k_chain: mode bytes (ChainDesc::byte_off)
    int entry = LWB_ENTRY_SPECTRUM;                         // k_chain: else its own front half on residues / VQ records
    const float *coeffs = nullptr, *dense = nullptr;
    const uint8_t *kinds = nullptr;
    const uint32_t *ys = nullptr;
    const float *zero = nullptr;                            // k_chain: curves of LWB_FLOOR_ZERO rows, or nullptr
    VqDev vq = {};                                          // k_chain, LWB_ENTRY_VQ: the batch's VQ arrays
    bool mix = false;                                       // k_chain: a chain's setup has an output mix
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
    bool floor0 = false;               // whether k_floor0_curves runs first (the packets may have LWB_FLOOR_ZERO rows)
};

struct lwb_plan {
    lwb_ctx *ctx = nullptr;
    lwb_chain *chains = nullptr;
    size_t n_chains = 0;
    lwb_batch_io io;
    // captured launch sequence (valid while ctx->state_gen == gen): the front stages if front.n, then `steps`.  Every
    // path that captures a residue-entry batch sets `front`; a spectrum-entry plan never does.
    bool captured = false;
    uint64_t gen = 0;
    FrontStages front;
    DevBuf pro, desc;                  // descriptors the capture owns: the long path's front stages, the steps'
    StepArgs args;
    std::vector<Step> steps;
};

struct lwb_stream {
    lwb_ctx *ctx = nullptr;
    const lwb_setup *setup = nullptr;
    float *d_state = nullptr;      // [channels][n1/2]
    bool has = false;              // PreviousWindowRight.data.is_some()
    uint32_t plen = 0;             // per-channel length of the saved right half
    uint64_t busy_epoch = 0;       // guards against one stream appearing twice in a batch
    uint64_t skip_left = 0;        // the output window (lwb_stream_set_window): samples still to drop ...
    uint64_t limit_left = ~0ull;   // ... and still to write after them (~0: no end)
};

// Records the launches a path made for a prepared batch; lwb_plan_execute replays them while ctx->state_gen == gen.
static void capture(lwb_plan *plan, uint64_t gen, const FrontStages &front, const StepArgs &args, std::vector<Step> steps)
{
    plan->captured = true;
    plan->gen = gen;
    plan->front = front;
    // Replays upload the host floor arrays of each step without looking at them: a later step may carry floor-0 records
    // that the captured one did not, so the floor-0 curves run whenever a chain's setup can serve records.
    for (size_t i = 0; i < plan->n_chains && front.n; i++)
        if (!plan->chains[i].stream->setup->floor0.empty()) plan->front.floor0 = true;
    plan->args = args;
    plan->steps = std::move(steps);
}


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

// Grows b to at least `bytes`.  The old buffer is freed once the last work that may use it has finished: the work
// before `in_use` when the arena belongs to a host set, else everything queued on the compute stream.
static int ensure(lwb_ctx *ctx, DevBuf &b, size_t bytes, cudaEvent_t in_use = nullptr)
{
    if (bytes <= b.cap) return LWB_OK;
    if (b.p) {
        if (in_use) CU(ctx, cudaEventSynchronize(in_use));
        else CU(ctx, cudaStreamSynchronize(ctx->stream));
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

// The next slot of the staging ring, at least `bytes` large, once the copy that last read it has finished.  A slot that
// grows keeps its old buffer until the context is destroyed: freeing it would wait for the whole device, other
// contexts' queued work included.  (Each growth at least doubles the slot, so the old buffers hold less than it does.)
static int acquire_staging(lwb_ctx *ctx, size_t bytes, Staging **out)
{
    Staging &st = ctx->stage[ctx->stage_next];
    ctx->stage_next = (ctx->stage_next + 1) % 3;
    if (!st.ev) CU(ctx, cudaEventCreateWithFlags(&st.ev, cudaEventDisableTiming));
    if (st.pending) {
        CU(ctx, cudaEventSynchronize(st.ev));      // waits for the descriptor copy only, not for kernels
        st.pending = false;
    }
    if (st.cap < bytes) {
        if (st.h) ctx->stage_old.push_back(st.h);
        st.h = nullptr;
        st.cap = 0;
        CU(ctx, cudaHostAlloc(&st.h, bytes * 2 + 4096, cudaHostAllocDefault));
        st.cap = bytes * 2 + 4096;
    }
    *out = &st;
    return LWB_OK;
}

// H2D of `bytes` from `src`, inside staging slot `st`, to `dst` on stream `s`; the slot is taken again behind this copy.
static int upload_staging(lwb_ctx *ctx, Staging *st, const void *src, void *dst, size_t bytes, cudaStream_t s)
{
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaEventRecord(st->ev, s));
    st->pending = true;
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
    for (ArenaSet &s : ctx->host_sets) CU(ctx, cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    return ensure(ctx, ctx->ticket, kTicketPool * sizeof(unsigned int));
}

// Retires tickets in order up to `upto`: the completed ones, or (block) all of them, waiting for each.
static int retire_tickets(lwb_ctx *ctx, uint64_t upto, bool block);

// Orders copy_out behind everything queued so far on copy_in and the compute stream, then records `set`'s `done`
// there (if given): what a set's next user waits for.
static int order_copy_out_behind_all(lwb_ctx *ctx, ArenaSet *set)
{
    CU(ctx, cudaEventRecord(ctx->ev_done[64], ctx->copy_in));
    CU(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_done[64], 0));
    CU(ctx, cudaEventRecord(ctx->ev_done[64], ctx->stream));
    CU(ctx, cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[64], 0));
    if (set) CU(ctx, cudaEventRecord(set->done, ctx->copy_out));
    return LWB_OK;
}

// Queues the completion ticket of the batch just queued: an event on copy_out behind the batch's last kernel and its
// last D2H.  `set`: the host set the batch used, whose `done` is recorded at the same point.  The ticket counts as
// issued only once its event is recorded.  Tickets that have completed are retired first (without waiting), so that
// a caller who never queries them does not accumulate events.
static int issue_ticket(lwb_ctx *ctx, ArenaSet *set)
{
    int rc;
    if ((rc = retire_tickets(ctx, ctx->tickets_issued, false)) || (rc = order_copy_out_behind_all(ctx, set))) return rc;
    cudaEvent_t ev;
    if (ctx->spare_events.empty()) {
        CU(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    } else {
        ev = ctx->spare_events.back();
        ctx->spare_events.pop_back();
    }
    const cudaError_t e = cudaEventRecord(ev, ctx->copy_out);
    if (e != cudaSuccess) {
        ctx->spare_events.push_back(ev);
        return fail(ctx, LWB_ERR_CUDA, "cudaEventRecord(ticket)", e);
    }
    ctx->ticket_events.push_back(ev);
    ctx->tickets_issued++;
    return LWB_OK;
}

static int retire_tickets(lwb_ctx *ctx, uint64_t upto, bool block)
{
    while (ctx->tickets_done < upto) {
        cudaEvent_t ev = ctx->ticket_events.front();
        const cudaError_t e = block ? cudaEventSynchronize(ev) : cudaEventQuery(ev);
        if (e == cudaErrorNotReady) {
            cudaGetLastError();
            return LWB_OK;
        }
        if (e != cudaSuccess) return fail(ctx, LWB_ERR_CUDA, "ticket", e);
        ctx->ticket_events.pop_front();
        ctx->spare_events.push_back(ev);
        ctx->tickets_done++;
    }
    return LWB_OK;
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

// f(std::integral_constant<int, fmt>()): how the kernels templated on an LWB_OUT_* value (k_chain, k_overlap) are picked
// for a runtime format.  Instantiated for every format out_format_known accepts.
template <int F = LWB_OUT_F32_PLANAR, typename Fn>
static int with_out_format(int fmt, Fn &&f)
{
    if constexpr (F > kOutFormatLast)
        return LWB_ERR_INVALID;
    else if constexpr (!out_format_known(F))
        return with_out_format<F + 1>(fmt, f);
    else
        return fmt == F ? f(std::integral_constant<int, F>()) : with_out_format<F + 1>(fmt, f);
}

// The layout the fused kernels take: planar out, and 16-byte aligned addresses, which their TMA bulk loads of
// coefficients and vector stores of PCM need.  Coefficient offsets that are multiples of 4 and PCM offsets that are
// multiples of the format's OutFormat::align (4; 16 for i24, whose 16 samples are 48 bytes) keep that when the arenas
// are 16-byte aligned: the library's staging of host-memory batches always is, a caller's device arena may not be (the
// chain kernel takes those).
static bool fused_layout(const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io)
{
    const OutFormat of = out_format_of(io->out_format);
    if (!of.planar) return false;
    if (io->memory == LWB_MEM_DEVICE && ((reinterpret_cast<uintptr_t>(io->coeffs) | reinterpret_cast<uintptr_t>(io->pcm) |
                                          reinterpret_cast<uintptr_t>(io->dense_floor)) & 15))
        return false;
    for (size_t i = 0; i < n_chains; i++)
        if (((chains[i].out_offset | chains[i].out_stride) & (of.align - 1)) || (chains[i].coeff_offset & 3)) return false;
    return true;
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

