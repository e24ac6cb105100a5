// path_mid.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// batches whose every packet is a full-window block of n = 1024 or of n = 512 (blocksize 10 / 9) go to k_mid
// (kernel_mid.cuh): planar f32 / i16, <= 8 channels; the residue entry runs the front stages (k_floor1_segments +
// k_prologue_fused, kernel_prologue.cuh) over all packets first and hand k_mid the spectrum arena.  The descriptors, the staging of host arenas and the capture by a prepared
// batch follow try_chain; the launch goes through mixed_launch_rounds (MixRound::nm).
#pragma once

struct MidGroup { LongRun r[4]; uint32_t n_packets; };

static int try_mid(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, uint64_t epoch, bool *handled,
                   lwb_plan *plan = nullptr)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (getenv("LWB_NO_MID")) return LWB_OK;
    if (io->out_format != LWB_OUT_F32_PLANAR && io->out_format != LWB_OUT_I16_PLANAR) return LWB_OK;
    const bool vq = io->entry == LWB_ENTRY_VQ, residue = io->entry != LWB_ENTRY_SPECTRUM;
    if (residue && !io->floor_kind) return LWB_OK;            // (the chain kernel words the error)
    if (vq) return LWB_OK;                                    // (VQ records of such streams: the general path, as before)
    if (!device_arenas_aligned(io)) return LWB_OK;
    int uniform_c = -1;
    const bool i16 = io->out_format == LWB_OUT_I16_PLANAR;
    const size_t esz = i16 ? 2 : 4;
    const float *pack = nullptr;
    int kb = 0;                                              // 1: n = 1024, 2: n = 512 (one size per batch: one pack)
    // pass 1, no side effects: every packet a full-window block of that size on top of no state or an n/2-sample one
    size_t n_runs = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        if (!c->stream || c->stream->ctx != ctx || (c->n_packets && !c->mode_numbers)) return LWB_OK;
        const lwb_setup *su = c->stream->setup;
        if (su->channels > 8 || (su->bs1 != 10 && su->bs1 != 9) || !su->host.tab[1].pack) return LWB_OK;
        if (residue) {                                        // the front stages want one channel count per batch
            if (uniform_c < 0) uniform_c = (int)su->channels;
            if (uniform_c != (int)su->channels) return LWB_OK;
        }
        if (pack && pack != su->host.tab[1].pack) return LWB_OK;
        pack = su->host.tab[1].pack;
        kb = 11 - su->bs1;
        if ((c->out_offset & 3) || (c->out_stride & 3) || (c->coeff_offset & 3)) return LWB_OK;
        const uint32_t n_blk = 2048u >> kb, n2_blk = n_blk >> 1;
        if (c->stream->has && c->stream->plen != n2_blk) return LWB_OK;
        for (uint32_t k = 0; k < c->n_packets; k++) {
            Geom g;
            if (geometry(su, c->mode_numbers[k], c->prev_window_flags ? c->prev_window_flags[k] : 1,
                         c->next_window_flags ? c->next_window_flags[k] : 1, &g))
                return LWB_OK;                                  // a bad mode number: the chain kernel reports it in place
            if (g.n != n_blk || g.ls != 0 || g.rs != n2_blk || g.re != n_blk) return LWB_OK;
        }
        if (c->n_packets) {
            // the planes hold the samples the chain produces: none for the first packet of an empty stream
            const uint64_t produced = (uint64_t)(c->n_packets - (c->stream->has ? 0u : 1u)) * n2_blk;
            if (c->out_stride < produced) return LWB_OK;     // (the chain kernel words the error)
            n_runs += su->channels;
        }
    }
    if (!pack || !n_runs) return LWB_OK;
    const size_t kMidN2 = 1024u >> kb, NBg = (size_t)1 << kb;
    *handled = true;

    const bool host = io->memory == LWB_MEM_HOST;
    cudaStream_t sm = ctx->stream;
    int rc;
    uint64_t c_lo = ~0ull, c_hi = 0, o_lo = ~0ull, o_hi = 0, r_lo = ~0ull, r_hi = 0;
    bool need_dense = false;
    size_t n_pk = 0;
    for (size_t i = 0; i < n_chains; i++) {
        lwb_chain *c = &chains[i];
        lwb_stream *s = c->stream;
        if (s->busy_epoch == epoch) return fail(ctx, LWB_ERR_INVALID, "a stream appears in two chains of one batch");
        s->busy_epoch = epoch;
        const unsigned C = s->setup->channels;
        if (residue && c->n_packets) {
            r_lo = std::min(r_lo, c->packet_index);
            r_hi = std::max<uint64_t>(r_hi, c->packet_index + c->n_packets);
            if ((rc = scan_floor_kinds(ctx, io, c->packet_index * C, (c->packet_index + c->n_packets) * C, &need_dense))) return rc;
            n_pk += c->n_packets;
        }
        c->status = LWB_OK;
        c->packets_done = c->n_packets;
        c->n_samples = c->n_packets ? (uint32_t)((c->n_packets - (s->has ? 0u : 1u)) * (uint32_t)kMidN2) : 0u;
        if (!c->n_packets) continue;
        c_lo = std::min(c_lo, c->coeff_offset);
        c_hi = std::max(c_hi, c->coeff_offset + (uint64_t)c->n_packets * C * kMidN2);
        o_lo = std::min(o_lo, c->out_offset);
        o_hi = std::max(o_hi, c->out_offset + (uint64_t)(C - 1) * c->out_stride + c->n_samples);
    }
    if (need_dense && !io->dense_floor) return fail(ctx, LWB_ERR_INVALID, "dense_floor missing");
    const float *d_coeffs = vq ? nullptr : io->coeffs;
    char *d_pcm = (char *)io->pcm;
    if (host) {
        if (o_hi > o_lo && (rc = ensure(ctx, ctx->pcm, (size_t)(o_hi - o_lo) * esz))) return rc;
        if (!vq) {
            if ((rc = ensure(ctx, ctx->coeffs, (size_t)(c_hi - c_lo) * 4))) return rc;
            CU(ctx, cudaMemcpyAsync(ctx->coeffs.p, io->coeffs + c_lo, (size_t)(c_hi - c_lo) * 4, cudaMemcpyHostToDevice, sm));
            d_coeffs = (const float *)ctx->coeffs.p - c_lo;
        }
        if (need_dense) {
            if ((rc = ensure(ctx, ctx->dense, (size_t)(c_hi - c_lo) * 4))) return rc;
            CU(ctx, cudaMemcpyAsync(ctx->dense.p, io->dense_floor + c_lo, (size_t)(c_hi - c_lo) * 4, cudaMemcpyHostToDevice, sm));
        }
        d_pcm = (char *)ctx->pcm.p - o_lo * esz;
    }
    // A prepared batch in device memory owns its descriptors (run groups, then the front stages' packet list) and replays
    // them while no stream changes shape (lwb_plan_execute).
    const bool capture = plan && !host;
    DevBuf &dbuf = capture ? plan->mix : ctx->cdesc;
    const size_t NBcap = (size_t)1 << kb;
    const size_t off_pro = (n_runs * NBcap * sizeof(LongRun) + 15) & ~(size_t)15;      // (an upper bound: every run its own group)
    if ((rc = ensure(ctx, dbuf, off_pro + n_pk * sizeof(DevPacket) + 16))) return rc;
    FrontStages fs;
    if (residue) {
        // front stages over every packet of the batch: residue (or VQ records) + floors -> spectrum arena, same element
        // offsets as the coefficient arena
        if ((rc = ensure(ctx, ctx->spec, (size_t)(c_hi - c_lo) * 4))) return rc;
        DevPacket *d_pro = (DevPacket *)((char *)dbuf.p + off_pro);
        fs.pk = d_pro;
        fs.n = n_pk;
        fs.C = (unsigned)uniform_c;
        fs.smem_old = prologue_smem(uniform_c, 11 - kb);
        fs.n2max = (int)kMidN2;
        fs.c_lo = c_lo;
        fs.r_lo = r_lo;
        fs.r_hi = r_hi;
        fs.dense = need_dense;
        Staging *stp;
        if ((rc = acquire_staging(ctx, n_pk * sizeof(DevPacket), &stp))) return rc;
        DevPacket *hp = (DevPacket *)stp->h;
        size_t di = 0;
        for (size_t i = 0; i < n_chains; i++) {
            write_front_packets(&chains[i], 0, chains[i].n_packets, chains[i].coeff_offset, hp + di);
            di += chains[i].n_packets;
        }
        fs.fast = front_stages_fast(ctx, io, fs, hp);
        CU(ctx, cudaMemcpyAsync(d_pro, hp, n_pk * sizeof(DevPacket), cudaMemcpyHostToDevice, sm));
        CU(ctx, cudaEventRecord(stp->ev, sm));
        stp->pending = true;
        if ((rc = front_stages_run(ctx, io, fs))) return rc;
        d_coeffs = (const float *)ctx->spec.p - c_lo;       // k_mid reads the spectrum
    }
    // runs, then groups of two runs of equal length (an odd one gets a dummy partner), longest first, dealt balanced
    std::vector<LongRun> runs;
    runs.reserve(n_runs);
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        if (!c->n_packets) continue;
        const lwb_stream *s = c->stream;
        const lwb_setup *su = s->setup;
        const unsigned C = su->channels;
        for (unsigned ch = 0; ch < C; ch++) {
            LongRun lr;
            std::memset(&lr, 0, sizeof(lr));
            lr.in = d_coeffs + c->coeff_offset + (size_t)ch * kMidN2;
            lr.out = d_pcm + (c->out_offset + (size_t)ch * c->out_stride) * esz;
            lr.state = s->d_state + (size_t)ch * state_stride(su);
            lr.in_stride = (uint32_t)(C * kMidN2);
            lr.n_packets = c->n_packets;
            lr.has_prev = s->has;
            lr.write_state = 1;
            runs.push_back(lr);
        }
    }
    std::stable_sort(runs.begin(), runs.end(), [](const LongRun &a, const LongRun &b) { return a.n_packets > b.n_packets; });
    std::vector<MidGroup> groups, tmp_g;
    groups.reserve(runs.size() / NBg + 8);
    for (size_t i = 0; i < runs.size();) {
        MidGroup g;
        std::memset(&g, 0, sizeof(g));
        g.n_packets = runs[i].n_packets;
        size_t k = 0;
        while (k < NBg && i < runs.size() && runs[i].n_packets == g.n_packets) g.r[k++] = runs[i++];
        for (; k < NBg; k++) {                    // dummies: read valid memory, store nothing
            g.r[k] = g.r[0];
            g.r[k].dummy = 1;
            g.r[k].write_state = 0;
            g.r[k].has_prev = 0;
        }
        groups.push_back(g);
    }
    const size_t Wg = std::min<size_t>((groups.size() + kLongWarps - 1) / kLongWarps, (size_t)ctx->sm_count) * kLongWarps;
    balance_static_deal(groups.data(), groups.size(), Wg, tmp_g);
    const size_t bytes = groups.size() * NBg * sizeof(LongRun);
    Staging *st;
    if ((rc = acquire_staging(ctx, bytes, &st))) return rc;
    LongRun *h = (LongRun *)st->h;
    for (size_t k = 0; k < groups.size(); k++)
        for (size_t b = 0; b < NBg; b++) h[NBg * k + b] = groups[k].r[b];
    if (bytes > off_pro) return fail(ctx, LWB_ERR_INVALID, "internal: more run groups than runs");
    CU(ctx, cudaMemcpyAsync(dbuf.p, h, bytes, cudaMemcpyHostToDevice, sm));
    CU(ctx, cudaEventRecord(st->ev, sm));
    st->pending = true;
    MixLaunch ml;
    std::memset(&ml, 0, sizeof(ml));
    ml.db = (char *)dbuf.p;
    ml.mpack = pack;
    ml.mid_kb = kb;
    ml.i16 = i16;
    ml.out_format = io->out_format;
    ml.pcm = d_pcm;
    MixRound rd;
    std::memset(&rd, 0, sizeof(rd));
    rd.nm = groups.size();
    std::vector<MixRound> rounds(1, rd);
    if ((rc = mixed_launch_rounds(ctx, ml, rounds))) return rc;
    if (capture) {
        plan->captured = true;
        plan->gen = gen_at_entry;
        plan->front = fs;                   // (no packets: spectrum entry)
        plan->mix_launch = ml;
        plan->mix_rounds = std::move(rounds);
    }
    if (host) {
        if (o_hi > o_lo && (rc = copy_pcm_to_host(ctx, io, chains, 0, n_chains, ctx->pcm.p, o_lo, sm))) return rc;
        CU(ctx, cudaStreamSynchronize(sm));
    }
    for (size_t i = 0; i < n_chains; i++)
        if (chains[i].n_packets) set_stream_state(chains[i].stream, true, (uint32_t)kMidN2);
    return LWB_OK;
}
