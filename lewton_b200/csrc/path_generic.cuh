// path_generic.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// per-packet planning of a batch and the four-kernel path (kernels_generic.cuh).
#pragma once

// ---------------------------------------------------------------------------------------------
// batch planning
// ---------------------------------------------------------------------------------------------
struct PlanPacket {
    Geom g;
    uint32_t plen;          // 0: no previous half -> 0 samples out
    uint64_t coeff_off;     // absolute element offset
    uint64_t sample_pos;    // samples (per channel) produced by the chain before this packet
};

struct PlanChain {
    lwb_chain *c;
    std::vector<PlanPacket> pk;
    bool end_has;           // stream state after the planned packets
    uint32_t end_plen;
    bool clear_after;       // OLA guard fired on packet pk.size(): state becomes empty
};

static int plan_chain(lwb_chain *c, PlanChain *pc)
{
    const lwb_stream *s = c->stream;
    const lwb_setup *su = s->setup;
    bool has = s->has;
    uint32_t plen = s->plen;
    uint64_t coeff = c->coeff_offset, pos = 0;
    pc->c = c;
    pc->clear_after = false;
    c->status = LWB_OK;
    pc->pk.reserve(c->n_packets);
    for (uint32_t i = 0; i < c->n_packets; i++) {
        PlanPacket pp;
        int rc = geometry(su, c->mode_numbers[i], c->prev_window_flags ? c->prev_window_flags[i] : 1,
                          c->next_window_flags ? c->next_window_flags[i] : 1, &pp.g);
        if (rc) { c->status = rc; break; }
        if (has) {
            const uint32_t slope_len = 1u << ((pp.g.slope_sel ? su->bs1 : su->bs0) - 1);
            if (slope_len < plen) {             // audio.rs:1107-1111; :1083 has already taken the state
                c->status = LWB_ERR_BAD_FORMAT;
                pc->clear_after = true;
                break;
            }
            if (pp.g.ls + plen > pp.g.n) {      // chan[range] would be out of bounds: a panic in the reference
                c->status = LWB_ERR_MISMATCH;
                break;
            }
        }
        pp.plen = has ? plen : 0;
        pp.coeff_off = coeff;
        pp.sample_pos = pos;
        coeff += (uint64_t)su->channels * (pp.g.n >> 1);
        if (has) pos += pp.g.rs - pp.g.ls;
        has = true;
        plen = pp.g.re - pp.g.rs;
        pc->pk.push_back(pp);
    }
    pc->end_has = pc->clear_after ? false : has;
    pc->end_plen = pc->clear_after ? 0 : plen;
    c->packets_done = (uint32_t)pc->pk.size();
    c->n_samples = (uint32_t)pos;
    return LWB_OK;
}

// dynamic shared memory k_prologue needs for the chains of a batch (curve bytes of the largest block)
static size_t prologue_smem_of(const std::vector<PlanChain> &plan)
{
    size_t m = 0;
    for (const PlanChain &pc : plan)
        if (pc.c && pc.c->stream) m = std::max(m, prologue_smem(pc.c->stream->setup->channels, pc.c->stream->setup->bs1));
    return m;
}

// Every launch of the library goes through launch() or launched(), which count it under its kernel's LWB_KERNEL_* id.
template <typename K, typename... Args>
static int launch(lwb_ctx *ctx, int kernel_id, K kernel, dim3 grid, dim3 block, size_t smem, Args... args)
{
    kernel<<<grid, block, smem, ctx->stream>>>(args...);
    count_launch(ctx, kernel_id);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, LWB_ERR_CUDA, "kernel launch", e);
    return LWB_OK;
}

// A launch made by a launch wrapper of the kernel headers (long_launch, mid_launch, short_launch, ...), which returns
// non-zero when it failed; `what` words the failure.
static int launched(lwb_ctx *ctx, int kernel_id, int wrapper_rc, const char *what)
{
    if (wrapper_rc) return fail(ctx, LWB_ERR_CUDA, what, cudaGetLastError());
    count_launch(ctx, kernel_id);
    return LWB_OK;
}

// Residue entry, front stages for `n_pk` packets of a batch with a uniform channel count C: spec[coeff_off ..] <-
// floor x inverse-coupled residue (audio.rs:991-1039).  The two-kernel form (kernel_prologue.cuh) needs <= 8
// channels and 16-byte aligned rows (prologue_is_fast); anything else takes the per-packet-CTA kernel.
static bool prologue_is_fast(const DevPacket *h_pk, size_t n_pk, unsigned C, const float *res, const float *dense, const float *spec)
{
    bool fast = C <= 8 && n_pk * (size_t)C < 0xffffffffu;
    for (size_t i = 0; fast && i < n_pk; i++) {
        const uint64_t e = h_pk[i].coeff_off;
        fast = (((res ? reinterpret_cast<uintptr_t>(res + e) : 0) | reinterpret_cast<uintptr_t>(spec + e) |
                 (dense ? reinterpret_cast<uintptr_t>(dense + e) : 0)) & 15) == 0 && h_pk[i].channels == C;
    }
    return fast;
}

// VQ views of a batch (LWB_ENTRY_VQ), device pointers biased like the floor arrays; runs == nullptr otherwise
struct VqView { const lwb_vq_run *runs = nullptr; const uint64_t *run_off = nullptr; const uint16_t *entries = nullptr; const uint64_t *ent_off = nullptr; };

// n2max: the largest n/2 among the packets (sizes the per-row bin -> segment index).
static int launch_prologue(lwb_ctx *ctx, const DevPacket *d_pk, size_t n_pk, unsigned C, bool fast, size_t smem_old, int n2max,
                           const float *res, const float *dense, const uint8_t *kinds, const uint32_t *ys, float *spec, VqView vq = VqView())
{
    if (!n_pk) return LWB_OK;
    const int words = std::max(1, (n2max + 31) >> 5);
    if (vq.runs && (!fast || (size_t)C * n2max > kVqMaxElems))
        return fail(ctx, LWB_ERR_INVALID, "VQ entry needs <= 8 channels, aligned arenas and channels * n/2 <= 12288");
    if (!fast)
        return launch(ctx, LWB_KERNEL_PROLOGUE, k_prologue, dim3((unsigned)n_pk), dim3(kPrologueThreads), smem_old, d_pk, res, dense, kinds, ys, spec);
    // per (packet, channel) row (ctx scratch): the packed flagged segments of its floor curve, the bin -> segment
    // index (bitmap + prefix counts) and the segment count
    const size_t rows = n_pk * C, tab_bytes = rows * kSegStride * sizeof(uint4), ix_bytes = rows * seg_index_stride(words);
    int rc = ensure(ctx, ctx->segtab, tab_bytes + ix_bytes + rows + 64);
    if (rc) return rc;
    if (!ctx->magic.p) {            // multiply-high magics of every segment length, once per context
        std::vector<uint32_t> mt(kFloor1MagicEntries);
        for (int adx = 0; adx < kFloor1MagicEntries; adx++) {
            int sh;
            mt[adx] = d_floor1_magic(adx, &sh);
        }
        if ((rc = ensure(ctx, ctx->magic, mt.size() * sizeof(uint32_t)))) return rc;
        CU(ctx, cudaMemcpy(ctx->magic.p, mt.data(), mt.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    uint4 *tab = (uint4 *)ctx->segtab.p;
    unsigned char *ix = (unsigned char *)ctx->segtab.p + tab_bytes;
    uint8_t *cnt = ix + ix_bytes;
    rc = launch(ctx, LWB_KERNEL_FLOOR1_SEGMENTS, k_floor1_segments, dim3((unsigned)((rows + kSegRows - 1) / kSegRows)), dim3(kSegThreads), floor1_segments_smem(words), d_pk,
                (uint32_t)rows, (int)C, kinds, ys, tab, cnt, ix, words, (const uint32_t *)ctx->magic.p);
    if (rc) return rc;
    const size_t grid = std::min<size_t>(n_pk, (size_t)ctx->sm_count * (C > 2 ? 4 : 8));
    const VqDev vd{vq.runs, vq.run_off, vq.entries, vq.ent_off};
    if (vq.runs)
        return launch(ctx, LWB_KERNEL_PROLOGUE_FUSED, k_prologue_fused<true>, dim3((unsigned)grid), dim3(kPfThreads), prologue_fused_smem((int)C, words, (size_t)C * n2max), d_pk,
                      (uint32_t)n_pk, res, dense, kinds, (const uint4 *)tab, (const uint8_t *)cnt, (const unsigned char *)ix, words, spec, vd);
    return launch(ctx, LWB_KERNEL_PROLOGUE_FUSED, k_prologue_fused<false>, dim3((unsigned)grid), dim3(kPfThreads), prologue_fused_smem((int)C, words), d_pk, (uint32_t)n_pk, res, dense,
                  kinds, (const uint4 *)tab, (const uint8_t *)cnt, (const unsigned char *)ix, words, spec, vd);
}
static int launch_prologue(lwb_ctx *ctx, const DevPacket *d_pk, const DevPacket *h_pk, size_t n_pk, unsigned C, size_t smem_old,
                           const float *res, const float *dense, const uint8_t *kinds, const uint32_t *ys, float *spec, VqView vq = VqView())
{
    int n2max = 32;
    for (size_t i = 0; i < n_pk; i++) n2max = std::max(n2max, h_pk[i].n >> 1);
    return launch_prologue(ctx, d_pk, n_pk, C, prologue_is_fast(h_pk, n_pk, C, res, dense, spec), smem_old, n2max, res, dense, kinds, ys, spec, vq);
}

// Host-side look at the floor kinds of rows [row_lo, row_hi) (one row per (packet, channel)).  Device-resident
// floor arrays (io->floor_memory == LWB_MEM_DEVICE) cannot be looked at: they are trusted, and the batch is assumed
// to carry dense (floor-0) curves exactly when the caller passed a dense_floor arena.
static int scan_floor_kinds(lwb_ctx *ctx, const lwb_batch_io *io, uint64_t row_lo, uint64_t row_hi, bool *need_dense)
{
    if (io->floor_memory == LWB_MEM_DEVICE) {
        if (io->dense_floor) *need_dense = true;
        return LWB_OK;
    }
    for (uint64_t r = row_lo; r < row_hi; r++) {
        const uint8_t kd = io->floor_kind[r];
        if (kd > LWB_FLOOR_DENSE) return fail(ctx, LWB_ERR_INVALID, "floor_kind out of range");
        if (kd == LWB_FLOOR_ONE && !io->floor1_y) return fail(ctx, LWB_ERR_INVALID, "floor1_y missing");
        if (kd == LWB_FLOOR_DENSE) *need_dense = true;
    }
    return LWB_OK;
}

// Device view of the floor arrays for packet rows [r_lo, r_hi) of a batch with C channels, biased so that ABSOLUTE
// row indices address them: host arrays are uploaded to ctx->kinds / ctx->ys on `sm`, device arrays are used in place.
static int stage_floor_arrays(lwb_ctx *ctx, const lwb_batch_io *io, uint64_t r_lo, uint64_t r_hi, unsigned C, cudaStream_t sm,
                              const uint8_t **d_kinds, const uint32_t **d_ys)
{
    *d_kinds = nullptr;
    *d_ys = nullptr;
    if (io->floor_memory == LWB_MEM_DEVICE) {
        *d_kinds = io->floor_kind;
        *d_ys = io->floor1_y;
        return LWB_OK;
    }
    if (r_hi <= r_lo) return LWB_OK;
    int rc;
    const size_t rows = (size_t)(r_hi - r_lo) * C;
    if ((rc = ensure(ctx, ctx->kinds, rows))) return rc;
    CU(ctx, cudaMemcpyAsync(ctx->kinds.p, io->floor_kind + r_lo * C, rows, cudaMemcpyHostToDevice, sm));
    *d_kinds = (const uint8_t *)ctx->kinds.p - r_lo * C;
    if (io->floor1_y) {
        if ((rc = ensure(ctx, ctx->ys, rows * LWB_MAX_POSTS * sizeof(uint32_t)))) return rc;
        CU(ctx, cudaMemcpyAsync(ctx->ys.p, io->floor1_y + r_lo * C * LWB_MAX_POSTS, rows * LWB_MAX_POSTS * sizeof(uint32_t),
                                cudaMemcpyHostToDevice, sm));
        *d_ys = (const uint32_t *)ctx->ys.p - r_lo * C * LWB_MAX_POSTS;
    }
    return LWB_OK;
}

// LWB_ENTRY_VQ: device view of the VQ runs / entries of packet rows [r_lo, r_hi), biased so that absolute rows and
// absolute offsets address it (host arrays are uploaded to ctx scratch on `sm`: four copies, all small).
static int stage_vq_arrays(lwb_ctx *ctx, const lwb_batch_io *io, uint64_t r_lo, uint64_t r_hi, cudaStream_t sm, VqView *out)
{
    *out = VqView();
    if (io->entry != LWB_ENTRY_VQ) return LWB_OK;
    if (io->floor_memory == LWB_MEM_DEVICE) {
        out->runs = io->vq_runs;
        out->run_off = io->vq_run_offsets;
        out->entries = io->vq_entries;
        out->ent_off = io->vq_entry_offsets;
        return LWB_OK;
    }
    if (r_hi <= r_lo) return LWB_OK;
    int rc;
    const uint64_t o_lo = io->vq_run_offsets[r_lo], o_hi = io->vq_run_offsets[r_hi];
    const uint64_t e_lo = io->vq_entry_offsets[r_lo], e_hi = io->vq_entry_offsets[r_hi];
    if (o_hi < o_lo || e_hi < e_lo) return fail(ctx, LWB_ERR_INVALID, "vq offsets must be non-decreasing");
    const size_t nrow = (size_t)(r_hi - r_lo) + 1, nrun = (size_t)(o_hi - o_lo), nent = (size_t)(e_hi - e_lo);
    const size_t b_off = nrow * sizeof(uint64_t), b_run = std::max<size_t>(nrun, 1) * sizeof(lwb_vq_run);
    if ((rc = ensure(ctx, ctx->vqoff, 2 * b_off)) || (rc = ensure(ctx, ctx->vqrec, b_run + std::max<size_t>(nent, 1) * sizeof(uint16_t) + 16))) return rc;
    char *d_off = (char *)ctx->vqoff.p, *d_rec = (char *)ctx->vqrec.p;
    CU(ctx, cudaMemcpyAsync(d_off, io->vq_run_offsets + r_lo, b_off, cudaMemcpyHostToDevice, sm));
    CU(ctx, cudaMemcpyAsync(d_off + b_off, io->vq_entry_offsets + r_lo, b_off, cudaMemcpyHostToDevice, sm));
    if (nrun) CU(ctx, cudaMemcpyAsync(d_rec, io->vq_runs + o_lo, nrun * sizeof(lwb_vq_run), cudaMemcpyHostToDevice, sm));
    if (nent) CU(ctx, cudaMemcpyAsync(d_rec + b_run, io->vq_entries + e_lo, nent * sizeof(uint16_t), cudaMemcpyHostToDevice, sm));
    out->run_off = (const uint64_t *)d_off - r_lo;
    out->ent_off = (const uint64_t *)(d_off + b_off) - r_lo;
    out->runs = (const lwb_vq_run *)d_rec - o_lo;
    out->entries = (const uint16_t *)(d_rec + b_run) - e_lo;
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// front stages of the fused paths (FrontStages)
// ---------------------------------------------------------------------------------------------
// Writes the front-stage descriptors of packets [p0, p0 + n) of chain c, packet p0 starting at element offset `coeff`:
// one DevPacket per packet, whatever its blocksize.  Returns the element offset behind the last one.
static uint64_t write_front_packets(const lwb_chain *c, uint32_t p0, uint32_t n, uint64_t coeff, DevPacket *out)
{
    const lwb_setup *su = c->stream->setup;
    for (uint32_t q = 0; q < n; q++) {
        const uint8_t mode = c->mode_numbers[p0 + q];
        const bool lng = su->host.mode_blockflag[mode] != 0;
        const uint32_t nq = 1u << (lng ? su->bs1 : su->bs0);
        DevPacket &d = out[q];
        std::memset(&d, 0, sizeof(d));
        d.setup = su->d_setup;
        d.coeff_off = coeff;
        d.pkt_index = c->packet_index + p0 + q;
        d.n = (uint16_t)nq;
        d.blockflag = lng;
        d.mapping = su->host.mode_mapping[mode];
        d.channels = su->channels;
        coeff += (uint64_t)su->channels * (nq >> 1);
    }
    return coeff;
}

// The arenas the front stages read and write, biased by fs.c_lo: the caller's residues and dense floors (device
// memory) or their staged copies in ctx->coeffs / ctx->dense (host memory), and ctx->spec.
struct FrontArenas { const float *res, *dense; float *spec; };
static FrontArenas front_arenas(lwb_ctx *ctx, const lwb_batch_io *io, const FrontStages &fs)
{
    const bool host = io->memory == LWB_MEM_HOST;
    FrontArenas a;
    a.res = io->entry == LWB_ENTRY_VQ ? nullptr : host ? (const float *)ctx->coeffs.p - fs.c_lo : io->coeffs;
    a.dense = !fs.dense ? nullptr : host ? (const float *)ctx->dense.p - fs.c_lo : io->dense_floor;
    a.spec = (float *)ctx->spec.p - fs.c_lo;
    return a;
}

// Whether the two-kernel form takes fs's packets (host copy h_pk of its list).
static bool front_stages_fast(lwb_ctx *ctx, const lwb_batch_io *io, const FrontStages &fs, const DevPacket *h_pk)
{
    const FrontArenas a = front_arenas(ctx, io, fs);
    return prologue_is_fast(h_pk, fs.n, fs.C, a.res, a.dense, a.spec);
}

// Packets [k0, k0 + n) of fs on floor / VQ views the caller has staged.
static int front_stages_launch(lwb_ctx *ctx, const lwb_batch_io *io, const FrontStages &fs, size_t k0, size_t n,
                               const uint8_t *kinds, const uint32_t *ys, const VqView &vq)
{
    const FrontArenas a = front_arenas(ctx, io, fs);
    return launch_prologue(ctx, fs.pk + k0, n, fs.C, fs.fast, fs.smem_old, fs.n2max, a.res, a.dense, kinds, ys, a.spec, vq);
}

// Stages the floor and VQ arrays of fs's packet rows on the compute stream (host arrays are uploaded, device arrays
// read in place) and launches the front stages over every packet of fs.
static int front_stages_run(lwb_ctx *ctx, const lwb_batch_io *io, const FrontStages &fs)
{
    const uint8_t *kinds;
    const uint32_t *ys;
    VqView vq;
    int rc;
    if ((rc = stage_floor_arrays(ctx, io, fs.r_lo, fs.r_hi, fs.C, ctx->stream, &kinds, &ys))) return rc;
    if ((rc = stage_vq_arrays(ctx, io, fs.r_lo, fs.r_hi, ctx->stream, &vq))) return rc;
    return front_stages_launch(ctx, io, fs, 0, fs.n, kinds, ys, vq);
}

struct DevArenas {
    const float *coeffs;      // device
    const float *dense;       // device or null
    const uint8_t *kinds;     // device or null
    const uint32_t *ys;       // device or null
    void *pcm;                // device
    uint64_t coeff_base;      // element offset that device coeffs[0] corresponds to
    uint64_t pcm_base;        // element offset that device pcm[0] corresponds to
    VqView vq;                // LWB_ENTRY_VQ
};

// Generic path: rounds of packets bounded by the IMDCT scratch.
static int run_generic(lwb_ctx *ctx, std::vector<PlanChain> &plan, const lwb_batch_io *io, const DevArenas &ar)
{
    size_t maxp = 0;
    for (auto &pc : plan) maxp = std::max(maxp, pc.pk.size());
    if (maxp == 0) return LWB_OK;
    // x elements of one "packet column" (packet i of every chain), to size the rounds
    std::vector<uint32_t> start(plan.size(), 0);
    const bool planar = is_planar(io->out_format);
    while (true) {
        // pick how many packets per chain go into this round
        size_t x_elems = 0, n_desc = 0, spec_lo = ~(size_t)0, spec_hi = 0;
        std::vector<uint32_t> take(plan.size(), 0);
        bool any = false;
        for (uint32_t step = 0;; step++) {
            size_t add = 0;
            bool more = false;
            for (size_t ci = 0; ci < plan.size(); ci++) {
                const uint32_t i = start[ci] + step;
                if (i < plan[ci].pk.size() && take[ci] == step) {
                    add += (size_t)plan[ci].c->stream->setup->channels * plan[ci].pk[i].g.n;
                    more = true;
                }
            }
            if (!more) break;
            if (x_elems && x_elems + add > ctx->x_cap_elems) break;
            for (size_t ci = 0; ci < plan.size(); ci++) {
                const uint32_t i = start[ci] + step;
                if (i < plan[ci].pk.size() && take[ci] == step) { take[ci]++; n_desc++; }
            }
            x_elems += add;
            any = true;
        }
        if (!any) break;
        int rc;
        if ((rc = ensure_pinned(ctx, n_desc * sizeof(DevPacket)))) return rc;
        if ((rc = ensure(ctx, ctx->desc, n_desc * sizeof(DevPacket)))) return rc;
        if ((rc = ensure(ctx, ctx->x, x_elems * sizeof(float)))) return rc;
        // the pinned descriptor staging is reused every round: wait for the previous upload
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        DevPacket *hp = (DevPacket *)ctx->h_desc;
        size_t di = 0, xo = 0;
        unsigned maxc = 1, maxn = 64;
        for (size_t ci = 0; ci < plan.size(); ci++) {
            PlanChain &pc = plan[ci];
            const lwb_stream *s = pc.c->stream;
            const lwb_setup *su = s->setup;
            const unsigned C = su->channels;
            for (uint32_t k = 0; k < take[ci]; k++) {
                const PlanPacket &pp = pc.pk[start[ci] + k];
                DevPacket &d = hp[di];
                std::memset(&d, 0, sizeof(d));
                d.setup = su->d_setup;
                d.state = s->d_state;
                d.coeff_off = pp.coeff_off - ar.coeff_base;
                d.x_off = xo;
                d.out_stride = pc.c->out_stride;
                d.out_off = pc.c->out_offset - ar.pcm_base + (planar ? pp.sample_pos : pp.sample_pos * C);
                d.pkt_index = pc.c->packet_index + start[ci] + k;
                d.prev_packet = k ? (int32_t)(di - 1) : -1;
                d.prev_rs = k ? hp[di - 1].rs : 0;
                d.state_stride = (uint32_t)state_stride(su);
                d.n = (uint16_t)pp.g.n;
                d.ls = (uint16_t)pp.g.ls;
                d.rs = (uint16_t)pp.g.rs;
                d.re = (uint16_t)pp.g.re;
                d.plen = (uint16_t)pp.plen;
                d.blockflag = pp.g.blockflag;
                d.mapping = pp.g.mapping;
                d.slope_sel = pp.g.slope_sel;
                d.channels = (uint8_t)C;
                d.save_state = (k + 1 == take[ci]);
                xo += (size_t)C * pp.g.n;
                spec_lo = std::min<size_t>(spec_lo, d.coeff_off);
                spec_hi = std::max<size_t>(spec_hi, d.coeff_off + (size_t)C * (pp.g.n >> 1));
                maxc = std::max(maxc, C);
                maxn = std::max<unsigned>(maxn, pp.g.n);
                di++;
            }
            start[ci] += take[ci];
        }
        CU(ctx, cudaMemcpyAsync(ctx->desc.p, hp, n_desc * sizeof(DevPacket), cudaMemcpyHostToDevice, ctx->stream));
        const DevPacket *dp = (const DevPacket *)ctx->desc.p;
        const float *spec = ar.coeffs;
        if (io->entry != LWB_ENTRY_SPECTRUM) {
            if ((rc = ensure(ctx, ctx->spec, spec_hi * sizeof(float)))) return rc;
            if ((rc = launch_prologue(ctx, dp, hp, n_desc, maxc, prologue_smem_of(plan), ar.coeffs, ar.dense, ar.kinds, ar.ys,
                                      (float *)ctx->spec.p, ar.vq)))
                return rc;
            spec = (const float *)ctx->spec.p;
        }
        if ((rc = launch(ctx, LWB_KERNEL_IMDCT, k_imdct, dim3((unsigned)n_desc, maxc), dim3(kImdctThreads), maxn * sizeof(float), dp,
                         spec, (float *)ctx->x.p)))
            return rc;
        dim3 g2((unsigned)n_desc, maxc), b2(kOverlapThreads);
        switch (io->out_format) {
        case LWB_OUT_F32_PLANAR: rc = launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<LWB_OUT_F32_PLANAR>, g2, b2, 0, dp, (const float *)ctx->x.p, ar.pcm); break;
        case LWB_OUT_I16_PLANAR: rc = launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<LWB_OUT_I16_PLANAR>, g2, b2, 0, dp, (const float *)ctx->x.p, ar.pcm); break;
        case LWB_OUT_F32_INTERLEAVED: rc = launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<LWB_OUT_F32_INTERLEAVED>, g2, b2, 0, dp, (const float *)ctx->x.p, ar.pcm); break;
        default: rc = launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<LWB_OUT_I16_INTERLEAVED>, g2, b2, 0, dp, (const float *)ctx->x.p, ar.pcm); break;
        }
        if (rc) return rc;
        if ((rc = launch(ctx, LWB_KERNEL_SAVE_STATE, k_save_state, g2, b2, 0, dp, (const float *)ctx->x.p))) return rc;
    }
    return LWB_OK;
}

