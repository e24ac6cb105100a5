// path_chain.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the chain-kernel path (kernel_chain.cuh), and the chain descriptors and row copies the mixed path shares with it.
#pragma once

// ---------------------------------------------------------------------------------------------
// Chain kernel path (kernel_chain.cuh): everything the fused long-block kernel does not take,
// as long as channels <= 8 and the per-channel buffers fit in shared memory.
// ---------------------------------------------------------------------------------------------
// Shared memory of the chain kernel: per channel `np` blocks of U | V plus the previous right half, the
// floor posts of up to 8 channels and, VQ entry, the residue accumulators (maxc * n1max / 2 floats: <= 48 KB within
// kVqMaxElems, 194 KB in all at most).  np (blocks a channel group transforms together) is 4 where that fits.
static size_t chain_smem(unsigned maxc, int n1max, int np, bool vq = false)
{
    return (size_t)maxc * ((size_t)np * n1max + n1max / 2) * 4 + 8 * (LWB_MAX_POSTS + 1) * 2 * 2 + 64 +
           (vq ? (size_t)maxc * (n1max / 2) * 4 : 0);
}
static int chain_np(unsigned maxc, int n1max, int wpc, bool residue)
{
    if (residue || wpc != 1) return 1;
    int np = 4;
    while (np > 1 && chain_smem(maxc, n1max, np) > 64 * 1024) np >>= 1;
    return np;
}
// k_chain for chains of up to maxc channels and blocks of up to n1max: one warp per channel and 1024 samples of the
// largest block, at most 32 warps per CTA.  residue: the residue or the VQ entry (vq).
static ChainShape chain_shape(unsigned maxc, int n1max, bool residue, bool vq = false)
{
    int wpc = std::max(1, std::min(8, n1max / 1024));
    while (wpc > 1 && (unsigned)wpc * maxc > 32) wpc >>= 1;
    const int np = chain_np(maxc, n1max, wpc, residue);
    return ChainShape{maxc * wpc, chain_smem(maxc, n1max, np, vq), n1max, wpc, np};
}

// One block per row: the stream state the first segment of a chain starts from, moved out of the way of the segment of
// the same chain that ends the batch -- in the one-pass schedule (path_mixed.cuh) that one may store the new state before
// the first one has read the old; and the state rows lwb_streams_save / lwb_streams_load move, whose offsets in the
// caller's buffer may leave a row unaligned or of a length that is not a multiple of 4; and the written samples of a
// clipped chain (BatchWalk::clip), rows of any sample type from its full output to their place -- at any byte alignment
// and of any byte length, as rows of 3-byte samples are.  Every row is stored in full 16-byte lines between a byte-wise
// head (up to dst's next 16-byte boundary) and a byte-wise tail, each under 16 bytes.  Where source and destination
// agree mod 16 the lines are plain vector copies; otherwise each line is funnel-shifted out of the two aligned 16-byte
// source lines it straddles (Q: its offset in words, r: the 0, 8, 16 or 24 bits left over).  Those lines hold at least
// one byte of the row each, so the loads stay inside the row's 16-byte lines.
template <int Q>
__device__ __forceinline__ void row_copy_shifted(const uint4 *__restrict__ a, uint4 *__restrict__ d, uint64_t nv, unsigned r)
{
    for (uint64_t v = threadIdx.x; v < nv; v += blockDim.x) {
        const uint4 A = a[v], B = a[v + 1];
        const uint32_t w[8] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w};
        d[v] = make_uint4(__funnelshift_r(w[Q], w[Q + 1], r), __funnelshift_r(w[Q + 1], w[Q + 2], r), __funnelshift_r(w[Q + 2], w[Q + 3], r),
                          __funnelshift_r(w[Q + 3], w[Q + 4], r));
    }
}

static_assert(kRowCopyThreads >= 16, "one thread per byte of a row's head and of its tail");
__global__ void __launch_bounds__(kRowCopyThreads) k_row_copy(const RowCopy *__restrict__ rc)
{
    const RowCopy c = rc[blockIdx.x];
    const char *src = static_cast<const char *>(c.src);
    char *dst = static_cast<char *>(c.dst);
    const uint64_t head = min(c.bytes, (uint64_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
    const uint64_t nv = (c.bytes - head) >> 4;
    if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
    if (head + nv * 16 + threadIdx.x < c.bytes) dst[head + nv * 16 + threadIdx.x] = src[head + nv * 16 + threadIdx.x];
    uint4 *d = reinterpret_cast<uint4 *>(dst + head);
    const char *s = src + head;
    const unsigned sh = reinterpret_cast<uintptr_t>(s) & 15, r = (sh & 3) * 8;
    const uint4 *a = reinterpret_cast<const uint4 *>(s - sh);
    switch (sh >> 2) {
    case 0:
        if (!sh) {
            for (uint64_t v = threadIdx.x; v < nv; v += blockDim.x) d[v] = a[v];
            return;
        }
        row_copy_shifted<0>(a, d, nv, r);
        return;
    case 1: row_copy_shifted<1>(a, d, nv, r); return;
    case 2: row_copy_shifted<2>(a, d, nv, r); return;
    default: row_copy_shifted<3>(a, d, nv, r); return;
    }
}

// The chain kernel's descriptor of packets [p0, p0 + n) of chain c, which enter with stream state (has, plen), start at
// element offset `coeff` and emit from sample `pos` of the chain's output; their mode bytes start at byte_off.
static void chain_desc(const lwb_chain *c, uint32_t p0, uint32_t n, bool has, uint32_t plen, uint64_t coeff, uint64_t pos, uint32_t byte_off,
                       ChainDesc *d)
{
    const lwb_stream *s = c->stream;
    const lwb_setup *su = s->setup;
    std::memset(d, 0, sizeof(*d));
    d->setup = su->d_setup;
    d->state = s->d_state;
    d->coeff_off = coeff;
    d->out_off = c->out_offset + pos;
    d->out_stride = c->out_stride;
    d->pkt_index = c->packet_index + p0;
    d->n_packets = n;
    d->byte_off = byte_off;
    d->state_stride = (uint32_t)state_stride(su);
    d->plen0 = (uint16_t)plen;
    d->has0 = has;
    d->channels = (uint8_t)su->channels;
}

// k_floor0_curves over the decoded packets of a residue- or VQ-entry batch the chain kernel takes: *zero addresses the curves by
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

static int try_chain(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled,
                     lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    const bool vq = io->entry == LWB_ENTRY_VQ, residue = io->entry != LWB_ENTRY_SPECTRUM;
    unsigned maxc = 1;
    int n1max = 64;
    size_t total_packets = 0;
    bool mix = false;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_setup *su = chains[i].stream->setup;
        if (su->channels > 8) return LWB_OK;
        mix |= su->host.n_out != 0;
        maxc = std::max<unsigned>(maxc, su->channels);
        n1max = std::max(n1max, 1 << su->bs1);
        total_packets += chains[i].n_packets;
    }
    // (VQ: the accumulators of the largest block; the four-kernel path words the error of a batch beyond them)
    if ((vq && (size_t)maxc * (n1max / 2) > kVqMaxElems) || chain_smem(maxc, n1max, 1, vq) > 200 * 1024) return LWB_OK;
    *handled = true;

    int rc;
    Staging *st;
    const size_t desc_bytes = n_chains * sizeof(ChainDesc), byte_bytes = total_packets * 3 + 16;
    if ((rc = acquire_staging(ctx, desc_bytes + byte_bytes, &st))) return rc;
    ChainDesc *hd = (ChainDesc *)st->h;
    uint8_t *hb = (uint8_t *)st->h + desc_bytes;
    const BatchExtent &ext = bw.ext;
    size_t boff = 0, n_launch = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const uint32_t done = bw.walks[i].done;
        if (!done) continue;
        for (uint32_t k = 0; k < done; k++) write_mode_bytes(c, k, hb + boff + 3 * k);
        chain_desc(c, 0, done, c->stream->has, c->stream->plen, c->coeff_offset, 0, (uint32_t)boff, &hd[n_launch++]);
        boff += (size_t)done * 3;
    }
    if (n_launch) {
        BatchArenas ar;
        if ((rc = ar.open(ctx, io, ext, maxc, false)) || (rc = ar.upload(0, ext))) return rc;
        cudaStream_t sm = ctx->stream;
        // descriptors and mode bytes share one device buffer; a prepared batch (device memory, spectrum
        // entry) owns it and replays the launch while no stream changes shape (residue and VQ entries are not captured)
        const bool cap = plan && !ar.host && !residue;
        DevBuf &dbuf = cap ? plan->desc : ctx->cdesc;
        const size_t used_desc = n_launch * sizeof(ChainDesc);
        if ((rc = ensure(ctx, dbuf, used_desc + boff + 16))) return rc;
        if ((rc = upload_staging(ctx, st, hd, dbuf.p, used_desc, sm)) ||
            (rc = upload_staging(ctx, st, hb, (char *)dbuf.p + used_desc, boff + 16, sm)))
            return rc;
        // residue or VQ entry with floor-0 records: their curves first, by absolute coefficient offset like ar.coeffs
        float *zero = nullptr;
        if (residue && ext.need_floor0 && ar.fl.ys && (rc = chain_floor0_curves(ctx, ar, ext, chains, n_chains, bw.walks, &zero))) return rc;
        StepArgs args;
        args.pcm = ar.pcm;
        args.out_format = io->out_format;
        args.chain = chain_shape(maxc, n1max, residue, vq);
        args.bytes = (const uint8_t *)dbuf.p + used_desc;
        args.entry = io->entry;
        args.coeffs = ar.coeffs;
        args.dense = ar.dense;
        args.kinds = ar.fl.kinds;
        args.ys = ar.fl.ys;
        args.zero = zero;
        args.vq = VqDev{ar.fl.vq.runs, ar.fl.vq.run_off, ar.fl.vq.entries, ar.fl.vq.ent_off};
        args.mix = mix;
        std::vector<Step> steps(1, Step{LWB_KERNEL_CHAIN, dbuf.p, n_launch, nullptr});
        if ((rc = run_steps(ctx, args, steps))) return rc;
        if (cap) capture(plan, gen_at_entry, FrontStages(), args, std::move(steps));
        if ((rc = ar.download(0, bw, 0, n_chains, ext)) || (rc = ar.finish())) return rc;
    }
    return LWB_OK;
}

