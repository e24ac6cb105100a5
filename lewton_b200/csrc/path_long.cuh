// path_long.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the fused long-block path (kernel_long.cuh): run cutting and descriptor staging, for the spectrum and the residue entries.
#pragma once

// ---------------------------------------------------------------------------------------------
// Fused path (kernel_long.cuh).  Eligible batches: spectrum entry, planar f32 out, every packet a
// long block of blocksize 2^11 with long neighbours, every stream either empty or holding a
// 1024-sample right half.  Planned directly from the chain list in O(chains + mode bytes) -- at
// 0.8 G blocks/s per GPU a per-packet host plan would be the bottleneck.
// ---------------------------------------------------------------------------------------------
struct LongItem {
    const lwb_chain *c;
    uint32_t P;
    bool has_prev;
};

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
        if (st.h) cudaFreeHost(st.h);
        st.h = nullptr;
        st.cap = 0;
        CU(ctx, cudaHostAlloc(&st.h, bytes * 2 + 4096, cudaHostAllocDefault));
        st.cap = bytes * 2 + 4096;
    }
    *out = &st;
    return LWB_OK;
}

// Appends the runs of one chain.  A chain (one channel of one stream) is cut into several runs
// when there are too few chains to fill the machine; every run after the first re-transforms the
// packet before its first one as a primer (its right half is all the run needs), which keeps
// runs independent at the cost of one extra IMDCT per cut.  coeffs / pcm: arenas addressed by absolute element offset.
static void long_runs_of(const LongItem &it, size_t cuts, const float *coeffs, char *pcm, size_t esz, LongRun *&w)
{
    const lwb_stream *s = it.c->stream;
    const lwb_setup *su = s->setup;
    const unsigned C = su->channels;
    const size_t P = it.P;
    for (unsigned ch = 0; ch < C; ch++) {
        const float *in0 = coeffs + it.c->coeff_offset + (size_t)ch * kLongN2;
        char *out0 = pcm + (it.c->out_offset + (size_t)ch * it.c->out_stride) * esz;
        for (size_t k = 0; k < cuts; k++) {
            const size_t p0 = P * k / cuts, p1 = P * (k + 1) / cuts;   // this run emits packets [p0, p1)
            LongRun &r = *w++;
            std::memset(&r, 0, sizeof(r));
            r.in_stride = (uint32_t)(C * kLongN2);
            r.state = s->d_state + (size_t)ch * state_stride(su);
            r.write_state = (k + 1 == cuts);
            if (k == 0) {
                r.in = in0;
                r.n_packets = (uint32_t)(p1 - p0);
                r.has_prev = it.has_prev;
                r.out = out0;
            } else {
                r.in = in0 + (p0 - 1) * (size_t)r.in_stride;           // primer = packet p0 - 1
                r.n_packets = (uint32_t)(p1 - p0 + 1);
                r.has_prev = 0;
                // samples emitted before packet p0: packets 0..p0-1, minus the first if no state
                r.out = out0 + (size_t)(p0 - (it.has_prev ? 0 : 1)) * kLongN2 * esz;
            }
        }
    }
}

// Every packet a long block of the fast blocksize with long neighbours, every stream empty or
// holding a 1024-sample right half, arenas aligned: what the fused kernel takes.
static bool batch_is_uniform_long(const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io)
{
    if (io->out_format != LWB_OUT_F32_PLANAR && io->out_format != LWB_OUT_I16_PLANAR) return false;
    const float *pack = nullptr;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_stream *s = c->stream;
        const lwb_setup *su = s->setup;
        if (su->bs1 != kLongBs || !su->host.tab[1].pack) return false;
        if (pack && pack != su->host.tab[1].pack) return false;
        pack = su->host.tab[1].pack;
        if ((c->out_offset & 3) || (c->out_stride & 3) || (c->coeff_offset & 3) || !device_arenas_aligned(io)) return false;
        if (s->has && s->plen != (uint32_t)kLongN2) return false;
        for (uint32_t k = 0; k < c->n_packets; k++) {
            const uint8_t m = c->mode_numbers[k];
            if (m >= su->n_modes || !su->host.mode_blockflag[m]) return false;
            if (c->prev_window_flags && !c->prev_window_flags[k]) return false;
            if (c->next_window_flags && !c->next_window_flags[k]) return false;
        }
    }
    return true;
}

// The result of every chain of a uniform long batch, in closed form: all its packets decode, and each emits 1024
// samples but the first of an empty stream.
static void set_long_results(lwb_chain *chains, size_t n_chains)
{
    for (size_t i = 0; i < n_chains; i++) {
        lwb_chain *c = &chains[i];
        c->status = LWB_OK;
        c->packets_done = c->n_packets;
        c->n_samples = c->n_packets ? (uint32_t)((c->n_packets - (c->stream->has ? 0 : 1)) * kLongN2) : 0;
    }
}

// Adds chains [i0, i1) of a uniform long batch, their results set, to `ext`.
static int long_extent(lwb_ctx *ctx, const lwb_batch_io *io, const lwb_chain *chains, size_t i0, size_t i1, BatchExtent *ext)
{
    int rc = LWB_OK;
    for (size_t i = i0; i < i1 && !rc; i++) {
        const lwb_chain *c = &chains[i];
        rc = ext->add(ctx, io, c, c->n_packets, c->coeff_offset + (uint64_t)c->n_packets * c->stream->setup->channels * kLongN2, c->n_samples);
    }
    return rc;
}

// The k_long runs of a batch, or of one slice of a residue batch, in pinned staging: chunk k launches runs
// [r0, r0 + nr) of chains [i0, i1); chunks without runs are left out.
struct LongRuns {
    struct Chunk { size_t r0, nr, i0, i1; };
    std::vector<Chunk> chunks;
    Staging *st = nullptr;
    LongRun *h = nullptr, *d = nullptr;
    size_t n = 0;
    int par = 0;                       // which half of the double-buffered descriptors (ctx->runs_buf) they take
    bool own = false;                  // in a prepared batch's own buffer rather than ctx->runs_buf[par]
};

// Builds the runs of chains [0, n_chains) for n_chunks launches; each launch should see >= target_runs runs.  `own`:
// the device buffer of a prepared batch, which keeps its runs for later executions (runs that read ctx->spec stay valid
// because growing any ctx arena bumps state_gen, see ensure()); else ctx->runs_buf.
static int long_build_runs(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, size_t n_chunks, const float *coeffs, char *pcm,
                           size_t esz, DevBuf *own, LongRuns *lr)
{
    std::vector<LongItem> items;
    items.reserve(n_chains);
    size_t chan_chains = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        items.push_back(LongItem{c, c->n_packets, c->stream->has});
        if (c->n_packets) chan_chains += c->stream->setup->channels;
    }
    const size_t warp_slots = (size_t)ctx->sm_count * kLongWarps * kLongNB;
    size_t target_runs = warp_slots * 4;                   // ~4 groups per warp evens out the tail
    if (const char *e = getenv("LWB_LONG_TARGET_RUNS")) target_runs = (size_t)atol(e);
    const size_t min_run = 8;                              // packets per run below which a cut costs > 12%
    int rc;
    // count runs
    std::vector<size_t> cuts(items.size(), 1);
    size_t total_runs = 0;
    for (size_t i = 0; i < items.size(); i++) {
        if (!items[i].P) { cuts[i] = 0; continue; }
        // per launch (chunk) the machine should see >= target_runs runs
        const size_t per_launch = std::max<size_t>(1, chan_chains / n_chunks);
        size_t k = 1;
        if (per_launch < target_runs) k = (target_runs + per_launch - 1) / per_launch;
        cuts[i] = std::max<size_t>(1, std::min(k, items[i].P / min_run));
        total_runs += cuts[i] * items[i].c->stream->setup->channels;
    }
    // the kernel takes groups of kLongNB runs of equal length; unpaired runs get a dummy partner
    const size_t cap_runs = total_runs * (kLongNB > 1 ? 2 : 1) + kLongNB;
    if ((rc = acquire_staging(ctx, cap_runs * sizeof(LongRun), &lr->st))) return rc;
    lr->par = ctx->runs_par;
    ctx->runs_par ^= 1;
    DevBuf &rb = own ? *own : ctx->runs_buf[lr->par];
    lr->own = own != nullptr;
    if ((rc = ensure(ctx, rb, cap_runs * sizeof(LongRun)))) return rc;
    lr->d = (LongRun *)rb.p;
    LongRun *h_runs = (LongRun *)lr->st->h, *w = h_runs;
    lr->h = h_runs;
    std::vector<LongRun> tmp;
    std::vector<uint32_t> order;
    for (size_t k = 0; k < n_chunks; k++) {
        const size_t i0 = items.size() * k / n_chunks, i1 = items.size() * (k + 1) / n_chunks;
        LongRun *w0 = w;
        // NB == 1: descriptors are written straight into the pinned staging; otherwise into a scratch
        // vector that is regrouped below
        size_t chunk_runs = 0;
        for (size_t i = i0; i < i1; i++)
            if (items[i].P) chunk_runs += cuts[i] * items[i].c->stream->setup->channels;
        LongRun *gen = w;
        if (kLongNB > 1) {
            tmp.resize(chunk_runs);
            gen = tmp.data();
        }
        for (size_t i = i0; i < i1; i++)
            if (items[i].P) long_runs_of(items[i], cuts[i], coeffs, pcm, esz, gen);
        if (!chunk_runs) continue;
        if (kLongNB == 1) {
            w = gen;
        } else {
            // group runs of equal packet count (consecutive channels of a stream already are)
            bool sorted = true;
            for (size_t i = 1; i < tmp.size() && sorted; i++) sorted = tmp[i].n_packets == tmp[0].n_packets;
            order.resize(tmp.size());
            for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
            if (!sorted)
                std::stable_sort(order.begin(), order.end(),
                                 [&](uint32_t a, uint32_t b) { return tmp[a].n_packets < tmp[b].n_packets; });
            size_t i = 0;
            while (i < order.size()) {
                size_t j = i;
                while (j < order.size() && tmp[order[j]].n_packets == tmp[order[i]].n_packets) j++;
                for (size_t q = i; q < j; q++) *w++ = tmp[order[q]];
                size_t fill = (kLongNB - (j - i) % kLongNB) % kLongNB;
                while (fill--) {
                    LongRun d = tmp[order[j - 1]];       // reads valid memory, stores nothing
                    d.dummy = 1;
                    d.write_state = 0;
                    d.has_prev = 0;
                    *w++ = d;
                }
                i = j;
            }
        }
        lr->chunks.push_back(LongRuns::Chunk{(size_t)(w0 - h_runs), (size_t)(w - w0), i0, i1});
    }
    lr->n = (size_t)(w - h_runs);
    return LWB_OK;
}

// One descriptor upload for all the runs, on `ds`, behind the kernel that last read this half of the double buffer.
// A prepared batch's own buffer has no halves: every launch queued so far may be one of its replays, which read that
// buffer and record no ev_kdone, so a re-plan's upload waits for all of them.
static int long_upload_runs(lwb_ctx *ctx, const LongRuns &lr, cudaStream_t ds)
{
    int rc;
    if (lr.own && ds != ctx->stream && (rc = order_copies_behind_compute(ctx))) return rc;
    CU(ctx, cudaStreamWaitEvent(ds, ctx->ev_kdone[lr.par], 0));
    CU(ctx, cudaMemcpyAsync(lr.d, lr.h, lr.n * sizeof(LongRun), cudaMemcpyHostToDevice, ds));
    CU(ctx, cudaEventRecord(ctx->ev_desc[lr.par], ds));
    CU(ctx, cudaEventRecord(lr.st->ev, ds));
    lr.st->pending = true;
    CU(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_desc[lr.par], 0));
    return LWB_OK;
}

// One k_long launch over n_groups groups of runs.
static int launch_long(lwb_ctx *ctx, const LongRun *runs, uint32_t n_groups, const float *pack, bool i16)
{
    unsigned int *ticket;
    int rc = next_ticket(ctx, &ticket);
    if (rc) return rc;
    return launched(ctx, LWB_KERNEL_LONG, long_launch(ctx->stream, runs, n_groups, pack, ticket, ctx->sm_count, i16), "long kernel launch");
}

static int try_long(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, bool *handled, lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (io->entry != LWB_ENTRY_SPECTRUM || !batch_is_uniform_long(chains, n_chains, io)) return LWB_OK;
    *handled = true;
    set_long_results(chains, n_chains);
    BatchExtent ext;
    int rc;
    if ((rc = long_extent(ctx, io, chains, 0, n_chains, &ext))) return rc;
    if (ext.empty()) return LWB_OK;
    const bool i16 = io->out_format == LWB_OUT_I16_PLANAR, host = io->memory == LWB_MEM_HOST;
    const float *pack = chains[0].stream->setup->host.tab[1].pack;          // one twiddle pack per launch
    // host memory: chunks of chains
    const size_t n_chunks = host ? host_chunks((size_t)(ext.c_hi - ext.c_lo) * 4, n_chains) : 1;
    const bool cap = plan && !host;
    BatchArenas ar;
    LongRuns lr;
    // (host memory: the runs go up on copy_in, ahead of the chunks' inputs; behind copy_out's PCM copies the kernels
    // would wait for the D2H of the batch before)
    if ((rc = ar.open(ctx, io, ext, 0, true)) ||
        (rc = long_build_runs(ctx, chains, n_chains, n_chunks, ar.coeffs, ar.pcm, i16 ? 2 : 4, cap ? &plan->runs : nullptr, &lr)) ||
        (rc = long_upload_runs(ctx, lr, host ? ctx->copy_in : ctx->copy_out)))
        return rc;
    for (size_t k = 0; k < lr.chunks.size(); k++) {
        const LongRuns::Chunk &ck = lr.chunks[k];
        BatchExtent ke;
        ke.scan = false;
        if ((rc = long_extent(ctx, io, chains, ck.i0, ck.i1, &ke)) || (rc = ar.upload(k, ke)) ||
            (rc = launch_long(ctx, lr.d + ck.r0, (uint32_t)(ck.nr / kLongNB), pack, i16)) ||
            (rc = ar.download(k, chains, ck.i0, ck.i1, ke)))
            return rc;
    }
    CU(ctx, cudaEventRecord(ctx->ev_kdone[lr.par], ctx->stream));
    if (cap) capture(plan, gen_at_entry, FrontStages(), MixLaunch{nullptr, nullptr, 0, i16, pack}, {}, (uint32_t)(lr.chunks[0].nr / kLongNB));
    if ((rc = ar.finish())) return rc;
    for (size_t i = 0; i < n_chains; i++)
        if (chains[i].n_packets) set_stream_state(chains[i].stream, true, kLongN2);
    return LWB_OK;
}

// Residue-entry batches whose every packet is a long block with long neighbours: the front stages
// (k_floor1_segments + k_prologue_fused, or k_prologue) form the spectrum on the device, the fused kernel does the
// rest.  Planned straight from the chain list like try_long (no per-packet PlanChain vectors); a prepared batch
// keeps the front-stage descriptors and, for device-memory batches, the fused kernel's runs, so that a replay
// is three launches with no host work (lwb_plan_execute).
static int try_long_residue(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, bool *handled, lwb_plan *plan)
{
    *handled = false;
    if (io->entry == LWB_ENTRY_SPECTRUM || !batch_is_uniform_long(chains, n_chains, io)) return LWB_OK;
    *handled = true;
    set_long_results(chains, n_chains);
    BatchExtent ext;
    int rc;
    if ((rc = long_extent(ctx, io, chains, 0, n_chains, &ext)) || (rc = ext.finish(ctx, io))) return rc;
    if (ext.empty()) return LWB_OK;
    const unsigned C = chains[0].stream->setup->channels;
    const bool i16 = io->out_format == LWB_OUT_I16_PLANAR, host = io->memory == LWB_MEM_HOST;
    const float *pack = chains[0].stream->setup->host.tab[1].pack;
    size_t n_pk = 0;
    for (size_t i = 0; i < n_chains; i++) n_pk += chains[i].n_packets;
    cudaStream_t sm = ctx->stream;
    if ((rc = ensure(ctx, ctx->spec, (size_t)(ext.c_hi - ext.c_lo) * 4))) return rc;
    BatchArenas ar;
    if ((rc = ar.open(ctx, io, ext, C, true))) return rc;
    FrontStages fs;
    fs.n = n_pk;
    fs.C = C;
    fs.smem_old = prologue_smem((int)C, kLongBs);
    fs.n2max = kLongN2;
    fs.c_lo = ext.c_lo;
    fs.r_lo = ext.r_lo;
    fs.r_hi = ext.r_hi;
    fs.dense = ext.need_dense;
    if (plan && plan->pro.p && plan->front.pk == plan->pro.p && plan->front.n == n_pk) {
        // a prepared batch re-planned (host memory: every execution): the packet list of the previous execution
        // depends only on the plan's chain and mode arrays
        fs.pk = plan->front.pk;
        fs.fast = plan->front.fast;
    } else {
        Staging *st;
        if ((rc = acquire_staging(ctx, n_pk * sizeof(DevPacket), &st))) return rc;
        DevBuf &db = plan ? plan->pro : ctx->desc;
        if ((rc = ensure(ctx, db, n_pk * sizeof(DevPacket)))) return rc;
        DevPacket *hp = (DevPacket *)st->h;
        size_t di = 0;
        for (size_t i = 0; i < n_chains; i++) {
            write_front_packets(&chains[i], 0, chains[i].n_packets, chains[i].coeff_offset, hp + di);
            di += chains[i].n_packets;
        }
        fs.pk = (const DevPacket *)db.p;
        fs.fast = front_stages_fast(ctx, ar, fs, hp);
        CU(ctx, cudaMemcpyAsync(db.p, hp, n_pk * sizeof(DevPacket), cudaMemcpyHostToDevice, sm));
        CU(ctx, cudaEventRecord(st->ev, sm));
        st->pending = true;
    }
    if (plan) plan->front = fs;
    const uint64_t gen = ctx->state_gen;
    const bool cap = plan && !host;
    // Host memory: slices of chains flow through three streams -- copy_in brings a slice's inputs (dense residues, or
    // VQ runs / entries, and its floor rows), the compute stream runs its front stages and the fused kernel, copy_out
    // takes its PCM home -- so that H2D, kernels and D2H of consecutive slices overlap (the link is duplex).  The
    // descriptor upload of a slice goes on copy_in: behind copy_out's PCM copies the next slice's kernels would wait
    // for the previous slice's D2H.
    const size_t n_sl = host ? host_chunks(n_pk * (size_t)C * kLongN2 * 4, n_chains) : 1;
    const float *spec = (const float *)ctx->spec.p - ext.c_lo;
    size_t pk0 = 0;
    for (size_t sl = 0; sl < n_sl; sl++) {
        const size_t i0 = n_chains * sl / n_sl, i1 = n_chains * (sl + 1) / n_sl;
        BatchExtent se;
        se.scan = false;
        if ((rc = long_extent(ctx, io, chains, i0, i1, &se))) return rc;
        if (se.empty()) continue;
        size_t npk = 0;
        for (size_t i = i0; i < i1; i++) npk += chains[i].n_packets;
        LongRuns lr;
        if ((rc = ar.upload(sl, se)) || (rc = front_stages_launch(ctx, ar, fs, pk0, npk)) ||
            (rc = long_build_runs(ctx, chains + i0, i1 - i0, 1, spec, ar.pcm, i16 ? 2 : 4, cap ? &plan->runs : nullptr, &lr)) ||
            (rc = long_upload_runs(ctx, lr, host ? ctx->copy_in : ctx->copy_out)) ||
            (rc = launch_long(ctx, lr.d, (uint32_t)(lr.n / kLongNB), pack, i16)) || (rc = ar.download(sl, chains, i0, i1, se)))
            return rc;
        CU(ctx, cudaEventRecord(ctx->ev_kdone[lr.par], sm));
        if (cap) capture(plan, gen, fs, MixLaunch{nullptr, nullptr, 0, i16, pack}, {}, (uint32_t)(lr.n / kLongNB));
        pk0 += npk;
    }
    if ((rc = ar.finish())) return rc;
    for (size_t i = 0; i < n_chains; i++)
        if (chains[i].n_packets) set_stream_state(chains[i].stream, true, kLongN2);
    return LWB_OK;
}
