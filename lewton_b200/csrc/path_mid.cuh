// path_mid.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// batches whose every packet is a full-window block of n = 1024 or of n = 512 (blocksize 10 / 9) go to k_mid
// (kernel_mid.cuh): planar f32 / i16 / f16, <= 8 channels; the residue and VQ entries run the front stages (k_floor1_segments +
// k_prologue_fused, kernel_prologue.cuh) over all packets first and hand k_mid the spectrum arena.  The descriptors, the staging of host arenas and the capture by a prepared
// batch (any entry) follow try_chain; the launch is one LWB_KERNEL_MID step.
#pragma once

static int try_mid(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled,
                   lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (getenv("LWB_NO_MID")) return LWB_OK;
    const bool residue = io->entry != LWB_ENTRY_SPECTRUM;     // residue or VQ entry: the front stages run first
    if (!fused_layout(chains, n_chains, io)) return LWB_OK;
    const size_t esz = out_format_of(io->out_format).esz;
    const float *pack = nullptr;
    int kb = 0;                                              // 1: n = 1024, 2: n = 512 (one size per batch: one pack)
    // every packet decodes, a full-window block of that size on top of no state or an n/2-sample one (a bad mode
    // number: the chain kernel reports it in place)
    size_t n_runs = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_setup *su = c->stream->setup;
        const ChainWalk &w = bw.walks[i];
        if (su->channels > 8 || (su->bs1 != 10 && su->bs1 != 9) || !su->host.tab[1].pack) return LWB_OK;
        // blocksize_0 == blocksize_1: short packets and the left slope of long ones after a short block read tab[0] (audio.rs:
        // 1048, 1059-1088), which k_mid's one pack holds only when both tables are the same (the context shares equal tables)
        if (su->bs0 == su->bs1 && su->host.tab[0].pack != su->host.tab[1].pack) return LWB_OK;
        if (pack && pack != su->host.tab[1].pack) return LWB_OK;
        pack = su->host.tab[1].pack;
        kb = 11 - su->bs1;
        const uint32_t n_blk = 2048u >> kb;
        if (c->stream->has && c->stream->plen != n_blk >> 1) return LWB_OK;
        if (w.done != c->n_packets || (w.done && w.full_n != n_blk)) return LWB_OK;
        if (w.done) n_runs += su->channels;
    }
    if (!pack || !n_runs) return LWB_OK;
    const size_t kMidN2 = 1024u >> kb, NBg = (size_t)1 << kb;
    const unsigned C = chains[0].stream->setup->channels;     // (residue entry: the batch's one channel count)
    *handled = true;

    const bool host = io->memory == LWB_MEM_HOST;
    int rc;
    const BatchExtent &ext = bw.ext;
    size_t n_pk = 0;
    if (residue)
        for (size_t i = 0; i < n_chains; i++) n_pk += chains[i].n_packets;
    BatchArenas ar;
    if ((rc = ar.open(ctx, io, ext, C, false)) || (rc = ar.upload(0, ext))) return rc;
    const float *d_coeffs = ar.coeffs;
    // A prepared batch in device memory owns its descriptors (run groups, then the front stages' packet list) and replays
    // them while no stream changes shape (lwb_plan_execute).
    const bool cap = plan && !host;
    DevBuf &dbuf = cap ? plan->desc : ctx->cdesc;
    const size_t off_pro = (n_runs * NBg * sizeof(LongRun) + 15) & ~(size_t)15;      // (an upper bound: every run its own group)
    if ((rc = ensure(ctx, dbuf, off_pro + n_pk * sizeof(DevPacket) + 16))) return rc;
    FrontStages fs;
    if (residue) {
        // front stages over every packet of the batch: residue (or VQ records) + floors -> spectrum arena, same element
        // offsets as the coefficient arena
        if ((rc = ensure(ctx, ctx->spec, (size_t)(ext.c_hi - ext.c_lo) * 4))) return rc;
        fs = front_stages_of(ext, C, (int)(2 * kMidN2), n_pk);
        if ((rc = stage_front_packets(ctx, ar, chains, n_chains, dbuf, off_pro, &fs)) || (rc = front_stages_launch(ctx, ar, fs, 0, fs.n)))
            return rc;
        d_coeffs = (const float *)ctx->spec.p - ext.c_lo;       // k_mid reads the spectrum
    }
    // runs, then groups of NBg runs of equal length (filled up with dummies), longest first, dealt balanced
    std::vector<LongRun> runs;
    runs.reserve(n_runs);
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        if (!c->n_packets) continue;
        for (unsigned ch = 0; ch < c->stream->setup->channels; ch++) {
            runs.emplace_back();
            channel_run(c, ch, kMidN2, d_coeffs + c->coeff_offset, ar.pcm, esz, c->n_packets, c->stream->has, 0, 1, &runs.back());
        }
    }
    // dummies: read valid memory, store nothing
    auto groups = group_runs<4>(runs, NBg, [](LongRun d) { d.dummy = 1; d.write_state = 0; d.has_prev = 0; return d; });
    balance_static_deal(groups.data(), groups.size(), kLongWarps, ctx->sm_count);
    const size_t bytes = groups.size() * NBg * sizeof(LongRun);
    Staging *st;
    if ((rc = acquire_staging(ctx, bytes, &st))) return rc;
    LongRun *h = (LongRun *)st->h;
    for (size_t k = 0; k < groups.size(); k++)
        for (size_t b = 0; b < NBg; b++) h[NBg * k + b] = groups[k].r[b];
    if (bytes > off_pro) return fail(ctx, LWB_ERR_INVALID, "internal: more run groups than runs");
    if ((rc = upload_staging(ctx, st, h, dbuf.p, bytes, ctx->stream))) return rc;
    StepArgs args;
    args.pcm = ar.pcm;
    args.out_format = io->out_format;
    args.mid_kb = kb;
    std::vector<Step> steps(1, Step{LWB_KERNEL_MID, dbuf.p, groups.size(), pack});
    if ((rc = run_steps(ctx, args, steps))) return rc;
    if (cap) capture(plan, gen_at_entry, fs, args, std::move(steps));
    if ((rc = ar.download(0, bw, 0, n_chains, ext))) return rc;
    return ar.finish();
}
