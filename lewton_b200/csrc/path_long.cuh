// path_long.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the fused long-block path (kernel_long.cuh): its runs and their staging, for the spectrum and the residue entries.
#pragma once

// ---------------------------------------------------------------------------------------------
// Fused path (kernel_long.cuh).  Eligible batches: any entry, planar f32 / i16 / f16 out, every packet a
// long block of blocksize 2^11 with long neighbours, every stream either empty or holding a
// 1024-sample right half.  Planned directly from the chain list in O(chains + mode bytes) -- at
// 0.8 G blocks/s per GPU a per-packet host plan would be the bottleneck.
// ---------------------------------------------------------------------------------------------
struct LongItem {
    const lwb_chain *c;
    uint32_t P;
    bool has_prev;
};

// Appends the runs of one chain, each channel cut into `cuts` pieces.  coeffs / pcm: arenas addressed by absolute
// element offset.
static void long_runs_of(const LongItem &it, size_t cuts, const float *coeffs, char *pcm, size_t esz, LongRun *&w)
{
    for (unsigned ch = 0; ch < it.c->stream->setup->channels; ch++, w += cuts)
        channel_run(it.c, ch, kLongN2, coeffs + it.c->coeff_offset, pcm, esz, it.P, it.has_prev, it.has_prev ? kLongN2 : 0, cuts, w);
}

// Every packet decodes, a long block of the fast blocksize between long neighbours, every stream empty or holding a
// 1024-sample right half, the fused kernels' layout: what the fused kernel takes.
static bool batch_is_uniform_long(const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw)
{
    if (!fused_layout(chains, n_chains, io)) return false;
    const float *pack = nullptr;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_stream *s = c->stream;
        const lwb_setup *su = s->setup;
        if (su->bs1 != kLongBs || !su->host.tab[1].pack) return false;
        if (pack && pack != su->host.tab[1].pack) return false;
        pack = su->host.tab[1].pack;
        if (s->has && s->plen != (uint32_t)kLongN2) return false;
        if (bw.walks[i].done != c->n_packets || !bw.walks[i].long_only) return false;
    }
    return true;
}

// The k_long runs of a batch in pinned staging: chunk k (chains [n_chains * k / n_chunks, n_chains * (k + 1) / n_chunks))
// launches runs [r0, r0 + nr).
struct LongRuns {
    struct Chunk { size_t r0, nr; };
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
        lr->chunks.push_back(LongRuns::Chunk{(size_t)(w0 - h_runs), (size_t)(w - w0)});
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
    if ((rc = upload_staging(ctx, lr.st, lr.h, lr.d, lr.n * sizeof(LongRun), ds))) return rc;
    CU(ctx, cudaEventRecord(ctx->ev_desc[lr.par], ds));
    CU(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_desc[lr.par], 0));
    return LWB_OK;
}

// The fused long-block path for all three entries.  A residue-entry batch (LWB_ENTRY_RESIDUE or LWB_ENTRY_VQ) runs
// the front stages (k_floor1_segments + k_prologue_fused, or k_prologue) over each chunk's packets first: they form its
// spectrum in ctx->spec, which k_long then reads instead of the coefficient arena.  Planned straight from the chain
// list (no per-packet PlanChain vectors).  A prepared batch keeps the front stages' packet list and, in device memory,
// the runs, so that a replay has no host work (lwb_plan_execute).  Host memory: chunks of chains flow through three
// streams -- copy_in brings a chunk's inputs (coefficients, or residues / VQ records and floor rows), the compute
// stream runs its kernels, copy_out takes its PCM home -- so that H2D, kernels and D2H of consecutive chunks overlap
// (the link is duplex).  The runs of all chunks are built while the first chunk's inputs copy and go up once, on
// copy_in behind those inputs: behind copy_out's PCM copies the kernels would wait for the D2H of the batch before.
static int try_long(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled,
                    lwb_plan *plan)
{
    *handled = false;
    if (!batch_is_uniform_long(chains, n_chains, io, bw)) return LWB_OK;
    *handled = true;
    const BatchExtent &ext = bw.ext;
    if (ext.empty()) return LWB_OK;
    int rc;
    const unsigned C = chains[0].stream->setup->channels;                  // (residue entries: the batch's one count)
    const bool residue = io->entry != LWB_ENTRY_SPECTRUM, host = io->memory == LWB_MEM_HOST;
    const float *pack = chains[0].stream->setup->host.tab[1].pack;          // one twiddle pack per launch
    const size_t n_chunks = host ? host_chunks((size_t)(ext.c_hi - ext.c_lo) * 4, n_chains) : 1;
    const bool cap = plan && !host;
    BatchArenas ar;
    if ((rc = ar.open(ctx, io, ext, C, true))) return rc;
    const float *in = ar.coeffs;
    FrontStages fs;
    if (residue) {
        size_t n_pk = 0;
        for (size_t i = 0; i < n_chains; i++) n_pk += chains[i].n_packets;
        if ((rc = ensure(ctx, ctx->spec, (size_t)(ext.c_hi - ext.c_lo) * 4))) return rc;
        fs = front_stages_of(ext, C, kLongN, n_pk);
        if (plan && plan->pro.p && plan->front.pk == plan->pro.p && plan->front.n == n_pk) {
            // a prepared batch re-planned (host memory: every execution): the packet list of the previous execution
            // depends only on the plan's chain and mode arrays
            fs.pk = plan->front.pk;
            fs.fast = plan->front.fast;
        } else if ((rc = stage_front_packets(ctx, ar, chains, n_chains, plan ? plan->pro : ctx->desc, 0, &fs))) {
            return rc;
        }
        if (plan) plan->front = fs;
        in = (const float *)ctx->spec.p - ext.c_lo;                         // same element offsets as the coefficients
    }
    StepArgs args;
    args.pcm = ar.pcm;
    args.out_format = io->out_format;
    std::vector<Step> steps;                                                // the k_long of one chunk
    LongRuns lr;
    uint64_t gen = 0;
    size_t pk0 = 0;
    for (size_t k = 0; k < n_chunks; k++) {
        const size_t i0 = n_chains * k / n_chunks, i1 = n_chains * (k + 1) / n_chunks;
        const BatchExtent ke = chunk_extent(io, chains, bw, i0, i1);
        if (ke.empty()) continue;
        size_t npk = 0;
        for (size_t i = i0; i < i1; i++) npk += chains[i].n_packets;
        if ((rc = ar.upload(k, ke)) || (residue && (rc = front_stages_launch(ctx, ar, fs, pk0, npk)))) return rc;
        if (!lr.d) {
            if ((rc = long_build_runs(ctx, chains, n_chains, n_chunks, in, ar.pcm, out_format_of(io->out_format).esz, cap ? &plan->desc : nullptr, &lr)) ||
                (rc = long_upload_runs(ctx, lr, host ? ctx->copy_in : ctx->copy_out)))
                return rc;
            gen = ctx->state_gen;                                           // every arena the capture points into is sized
        }
        steps.assign(1, Step{LWB_KERNEL_LONG, lr.d + lr.chunks[k].r0, lr.chunks[k].nr / kLongNB, pack});
        if ((rc = run_steps(ctx, args, steps)) || (rc = ar.download(k, bw, i0, i1, ke))) return rc;
        pk0 += npk;
    }
    CU(ctx, cudaEventRecord(ctx->ev_kdone[lr.par], ctx->stream));
    if (cap) capture(plan, gen, fs, args, std::move(steps));                 // (one chunk)
    return ar.finish();
}
