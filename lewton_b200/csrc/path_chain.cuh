// path_chain.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the chain-kernel path (kernel_chain.cuh) and the launch sequence shared with the mixed path.
#pragma once

// ---------------------------------------------------------------------------------------------
// Chain kernel path (kernel_chain.cuh): everything the fused long-block kernel does not take,
// as long as channels <= 8 and the per-channel buffers fit in shared memory.
// ---------------------------------------------------------------------------------------------
// Shared memory of the chain kernel: per channel `np` blocks of U | V plus the previous right half, and the
// floor posts of up to 8 channels.  np (blocks a channel group transforms together) is 4 where that fits.
static size_t chain_smem(unsigned maxc, int n1max, int np)
{
    return (size_t)maxc * ((size_t)np * n1max + n1max / 2) * 4 + 8 * (LWB_MAX_POSTS + 1) * 2 * 2 + 64;
}
static int chain_np(unsigned maxc, int n1max, int wpc, bool residue)
{
    if (residue || wpc != 1) return 1;
    int np = 4;
    while (np > 1 && chain_smem(maxc, n1max, np) > 64 * 1024) np >>= 1;
    return np;
}
// k_chain for chains of up to maxc channels and blocks of up to n1max: one warp per channel and 1024 samples of the
// largest block, at most 32 warps per CTA
static ChainShape chain_shape(unsigned maxc, int n1max, bool residue)
{
    int wpc = std::max(1, std::min(8, n1max / 1024));
    while (wpc > 1 && (unsigned)wpc * maxc > 32) wpc >>= 1;
    const int np = chain_np(maxc, n1max, wpc, residue);
    return ChainShape{maxc * wpc, chain_smem(maxc, n1max, np), n1max, wpc, np};
}

template <int ENTRY>
static int launch_chain(lwb_ctx *ctx, int fmt, unsigned n_chains, unsigned warps, size_t smem, const ChainDesc *d,
                        const uint8_t *bytes, const float *coeffs, const float *dense, const uint8_t *kinds,
                        const uint32_t *ys, void *pcm, int n1max, int wpc, int np, const float *zero)
{
#define LWB_CHAIN_CASE(F)                                                                                    \
    case F:                                                                                                  \
        if (wpc == 1) {                                                                                      \
            cudaFuncSetAttribute(k_chain<F, ENTRY, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            return launch(ctx, LWB_KERNEL_CHAIN, k_chain<F, ENTRY, false>, dim3(n_chains), dim3(warps * 32), smem, d, bytes, coeffs, dense, \
                          kinds, ys, pcm, n1max, wpc, np, zero);                                              \
        }                                                                                                    \
        cudaFuncSetAttribute(k_chain<F, ENTRY, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        return launch(ctx, LWB_KERNEL_CHAIN, k_chain<F, ENTRY, true>, dim3(n_chains), dim3(warps * 32), smem, d, bytes, coeffs, dense, kinds, \
                      ys, pcm, n1max, wpc, 1, zero);
    switch (fmt) {
        LWB_CHAIN_CASE(LWB_OUT_F32_PLANAR)
        LWB_CHAIN_CASE(LWB_OUT_I16_PLANAR)
        LWB_CHAIN_CASE(LWB_OUT_F32_INTERLEAVED)
        LWB_CHAIN_CASE(LWB_OUT_I16_INTERLEAVED)
    }
#undef LWB_CHAIN_CASE
    return LWB_ERR_INVALID;
}

// one launch of the fused kernel and one of the chain kernel per round, in stream order
// One block per row: the stream state the first segment of a chain starts from, moved out of the way of the segment of
// the same chain that ends the batch -- in the one-pass schedule (path_mixed.cuh) that one may store the new state before
// the first one has read the old.
__global__ void k_row_copy(const RowCopy *__restrict__ rc)
{
    const RowCopy c = rc[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < c.n4; i += blockDim.x)
        reinterpret_cast<float4 *>(c.dst)[i] = reinterpret_cast<const float4 *>(c.src)[i];
}

static int mixed_launch_rounds(lwb_ctx *ctx, const MixLaunch &ml, const std::vector<MixRound> &rounds)
{
    cudaStream_t sm = ctx->stream;
    int rc = LWB_OK;
    for (const MixRound &rd : rounds) {
        if (rd.nm &&             // uniform 1024-point batches (path_mid.cuh)
            (rc = launched(ctx, LWB_KERNEL_MID, mid_launch(sm, (const LongRun *)ml.db, (uint32_t)rd.nm, ml.mpack, ctx->sm_count, ml.i16, ml.mid_kb),
                           "mid kernel launch")))
            return rc;
        if (rd.nx && (rc = launch(ctx, LWB_KERNEL_ROW_COPY, k_row_copy, dim3((unsigned)rd.nx), dim3(64), 0, (const RowCopy *)(ml.db + ml.off_rc) + rd.x0)))
            return rc;
        if (rd.nr) {
            unsigned int *ticket;
            if ((rc = next_ticket(ctx, &ticket))) return rc;
            if (kLongNB != 1) return fail(ctx, LWB_ERR_INVALID, "mixed path needs one run per warp");
            // one pass over many short runs: the static deal with its deeper lookahead (k_long_s); rounds: tickets
            if (rd.flat)
                rc = launched(ctx, LWB_KERNEL_LONG_S,
                              long_launch_static(sm, (const LongRun *)ml.db + rd.r0, (uint32_t)rd.nr, ml.pack, ctx->sm_count, ml.i16, ml.w_short, ml.ls),
                              "long kernel launch");
            else
                rc = launched(ctx, LWB_KERNEL_LONG,
                              long_launch(sm, (const LongRun *)ml.db + rd.r0, (uint32_t)rd.nr, ml.pack, ticket, ctx->sm_count, ml.i16, ml.w_short, ml.ls),
                              "long kernel launch");
            if (rc) return rc;
        }
        if (rd.ns &&
            (rc = launched(ctx, LWB_KERNEL_SHORT, short_launch(sm, (const ShortRun *)(ml.db + ml.off_sr) + rd.s0, (uint32_t)rd.ns, ml.spack, ctx->sm_count, ml.i16),
                           "short kernel launch")))
            return rc;
        if (rd.ng &&             // bursts: eight short runs of equal length per warp (k_short_g)
            (rc = launched(ctx, LWB_KERNEL_SHORT_G,
                           short_launch_groups(sm, (const ShortRun *)(ml.db + ml.off_sg) + rd.g0 * kShortOct, (uint32_t)rd.ng, ml.spack, ctx->sm_count, ml.i16),
                           "short burst kernel launch")))
            return rc;
        if (rd.nc) {
            const ChainDesc *dcd = (const ChainDesc *)(ml.db + ml.off_cd) + rd.c0;
            const uint8_t *dby = (const uint8_t *)(ml.db + ml.off_by);
            if (ml.residue)
                rc = launch_chain<LWB_ENTRY_RESIDUE>(ctx, ml.out_format, (unsigned)rd.nc, ml.chain.warps, ml.chain.smem, dcd, dby, ml.coeffs, ml.dense,
                                                     ml.kinds, ml.ys, ml.pcm, ml.chain.n1max, ml.chain.wpc, ml.chain.np, ml.zero);
            else
                rc = launch_chain<LWB_ENTRY_SPECTRUM>(ctx, ml.out_format, (unsigned)rd.nc, ml.chain.warps, ml.chain.smem, dcd, dby, ml.coeffs, ml.dense,
                                                      ml.kinds, ml.ys, ml.pcm, ml.chain.n1max, ml.chain.wpc, ml.chain.np, ml.zero);
            if (rc) return rc;
        }
    }
    return LWB_OK;
}

// k_floor0_curves over the decoded packets of a residue-entry batch the chain kernel takes: *zero addresses the curves by
// absolute coefficient offset.  The packet list goes to ctx->desc, which only work queued on the compute stream uses.
static int chain_floor0_curves(lwb_ctx *ctx, const BatchArenas &ar, const BatchExtent &ext, const lwb_chain *chains, size_t n_chains,
                               const std::vector<ChainWalk> &walks, float **zero)
{
    size_t n_pk = 0;
    for (size_t i = 0; i < n_chains; i++) n_pk += walks[i].done;
    Staging *st;
    int rc;
    if ((rc = acquire_staging(ctx, n_pk * sizeof(DevPacket), &st)) || (rc = ensure(ctx, ctx->desc, n_pk * sizeof(DevPacket))) ||
        (rc = ensure(ctx, ctx->floor0, (size_t)(ext.c_hi - ext.c_lo) * sizeof(float))))
        return rc;
    DevPacket *hp = (DevPacket *)st->h, *w = hp;
    for (size_t i = 0; i < n_chains; i++) {
        write_front_packets(&chains[i], 0, walks[i].done, chains[i].coeff_offset, w);
        w += walks[i].done;
    }
    if ((rc = upload_staging(ctx, st, hp, ctx->desc.p, n_pk * sizeof(DevPacket), ctx->stream))) return rc;
    *zero = (float *)ctx->floor0.p - ext.c_lo;
    return launch_floor0_curves(ctx, (const DevPacket *)ctx->desc.p, n_pk, ar.C, ar.fl.kinds, ar.fl.ys, *zero);
}

static int try_chain(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, bool *handled, lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (io->entry == LWB_ENTRY_VQ) return LWB_OK;            // (its residue stage runs inside the kernel, on dense vectors)
    const bool residue = io->entry == LWB_ENTRY_RESIDUE;
    unsigned maxc = 1;
    int n1max = 64;
    size_t total_packets = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_setup *su = chains[i].stream->setup;
        if (su->channels > 8) return LWB_OK;
        maxc = std::max<unsigned>(maxc, su->channels);
        n1max = std::max(n1max, 1 << su->bs1);
        total_packets += chains[i].n_packets;
    }
    if (chain_smem(maxc, n1max, 1) > 200 * 1024) return LWB_OK;
    *handled = true;

    int rc;
    Staging *st;
    const size_t desc_bytes = n_chains * sizeof(ChainDesc), byte_bytes = total_packets * 3 + 16;
    if ((rc = acquire_staging(ctx, desc_bytes + byte_bytes, &st))) return rc;
    ChainDesc *hd = (ChainDesc *)st->h;
    uint8_t *hb = (uint8_t *)st->h + desc_bytes;
    BatchExtent ext;
    size_t boff = 0, n_launch = 0;
    std::vector<ChainWalk> walks(n_chains);
    for (size_t i = 0; i < n_chains; i++) {
        lwb_chain *c = &chains[i];
        const lwb_stream *s = c->stream;
        const lwb_setup *su = s->setup;
        const ChainWalk &w = walks[i] = walk_chain(c, [&](uint32_t k, const Geom &, bool, uint32_t, uint64_t, uint64_t) {
            write_mode_bytes(c, k, hb + boff + 3 * k);
        });
        set_chain_result(c, w);
        if ((rc = ext.add(ctx, io, c, w.done, w.coeff_end, w.n_samples))) return rc;
        if (!w.done) continue;
        ChainDesc &d = hd[n_launch++];
        std::memset(&d, 0, sizeof(d));
        d.setup = su->d_setup;
        d.state = s->d_state;
        d.coeff_off = c->coeff_offset;
        d.out_off = c->out_offset;
        d.out_stride = c->out_stride;
        d.pkt_index = c->packet_index;
        d.n_packets = w.done;
        d.byte_off = (uint32_t)boff;
        d.state_stride = (uint32_t)state_stride(su);
        d.plen0 = (uint16_t)s->plen;
        d.has0 = s->has;
        d.channels = (uint8_t)su->channels;
        boff += (size_t)w.done * 3;
    }
    if ((rc = ext.finish(ctx, io))) return rc;
    if (n_launch) {
        BatchArenas ar;
        if ((rc = ar.open(ctx, io, ext, maxc, false)) || (rc = ar.upload(0, ext))) return rc;
        cudaStream_t sm = ctx->stream;
        // descriptors and mode bytes share one device buffer; a prepared batch (device memory, spectrum
        // entry) owns it and replays the launch while no stream changes shape
        const bool cap = plan && !ar.host && !residue;
        DevBuf &dbuf = cap ? plan->mix : ctx->cdesc;
        const size_t used_desc = n_launch * sizeof(ChainDesc);
        if ((rc = ensure(ctx, dbuf, used_desc + boff + 16))) return rc;
        if ((rc = upload_staging(ctx, st, hd, dbuf.p, used_desc, sm)) ||
            (rc = upload_staging(ctx, st, hb, (char *)dbuf.p + used_desc, boff + 16, sm)))
            return rc;
        // residue entry with floor-0 records: their curves first, by absolute coefficient offset like ar.coeffs
        float *zero = nullptr;
        if (residue && ext.need_floor0 && ar.fl.ys && (rc = chain_floor0_curves(ctx, ar, ext, chains, n_chains, walks, &zero))) return rc;
        const MixLaunch ml{(char *)dbuf.p, ar.pcm, io->out_format, false, nullptr, 0, nullptr, nullptr, nullptr, 0, 0, 0, used_desc, 0, 0,
                           residue, chain_shape(maxc, n1max, residue), ar.coeffs, ar.dense, ar.fl.kinds, ar.fl.ys, zero};
        std::vector<MixRound> rounds(1, MixRound{0, 0, 0, 0, 0, n_launch});
        if ((rc = mixed_launch_rounds(ctx, ml, rounds))) return rc;
        if (cap) capture(plan, gen_at_entry, FrontStages(), ml, std::move(rounds));
        if ((rc = ar.download(0, chains, 0, n_chains, ext)) || (rc = ar.finish())) return rc;
    }
    commit_stream_states(chains, walks);
    return LWB_OK;
}

