// path_generic.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// the chain walk, run helpers, extent and host-memory pipeline every batch path shares, and the four-kernel path (kernels_generic.cuh).
#pragma once

// ---------------------------------------------------------------------------------------------
// batch planning
// ---------------------------------------------------------------------------------------------
// What one chain decodes: the packets up to the first with a bad mode or an overlap the reference refuses, the samples
// they produce and the stream state they leave (audio.rs:1056-1073, 1083-1154).
struct ChainWalk {
    uint32_t done = 0;            // packets decoded
    int status = LWB_OK;
    uint64_t n_samples = 0;       // per channel
    uint64_t skip = 0;            // the stream's window (clip_to_window): of those samples, the first `skip` are dropped
    uint64_t written = 0;         // and the next `written` written (== n_samples without a window)
    bool end_has = false;         // stream state after them
    uint32_t end_plen = 0;
    bool clear_after = false;     // the OLA guard fired on packet `done`: the state becomes empty
    uint64_t coeff_end = 0;       // element offset behind the last decoded packet
    uint32_t full_n = 0;          // n of every decoded packet when all are full-window blocks of one size, else 0
    bool long_only = true;        // every decoded packet a long block between long neighbours (both window flags set)
    bool clipped() const { return skip || written != n_samples; }
};

// Walks chain c from its stream's state, with no side effects.  on_packet(k, g, has, plen, coeff, pos) sees every packet
// that decodes: its geometry, the state entering it, its coefficient offset and the samples the chain produced before it.
template <typename F>
static ChainWalk walk_chain(const lwb_chain *c, F &&on_packet)
{
    const lwb_setup *su = c->stream->setup;
    ChainWalk w;
    bool has = c->stream->has;
    uint32_t plen = c->stream->plen;
    uint64_t coeff = c->coeff_offset, pos = 0;
    for (uint32_t k = 0; k < c->n_packets; k++) {
        const int pf = c->prev_window_flags ? c->prev_window_flags[k] : 1, nf = c->next_window_flags ? c->next_window_flags[k] : 1;
        Geom g;
        const int rc = geometry(su, c->mode_numbers[k], pf, nf, &g);
        if (rc) { w.status = rc; break; }
        if (has) {
            const uint32_t slope_len = 1u << ((g.slope_sel ? su->bs1 : su->bs0) - 1);
            if (slope_len < plen) {             // audio.rs:1107-1111; :1083 has already taken the state
                w.status = LWB_ERR_BAD_FORMAT;
                w.clear_after = true;
                break;
            }
            if (g.ls + plen > g.n) {            // chan[range] would be out of bounds: a panic in the reference
                w.status = LWB_ERR_MISMATCH;
                break;
            }
        }
        on_packet(k, g, has, plen, coeff, pos);
        w.full_n = g.ls == 0 && g.rs == g.n >> 1 && g.re == g.n && (!w.done || w.full_n == g.n) ? g.n : 0;
        w.long_only = w.long_only && g.blockflag && pf && nf;
        coeff += (uint64_t)su->channels * (g.n >> 1);
        if (has) pos += g.rs - g.ls;
        has = true;
        plen = g.re - g.rs;
        w.done++;
    }
    w.n_samples = pos;
    w.end_has = !w.clear_after && has;
    w.end_plen = w.clear_after ? 0 : plen;
    w.coeff_end = coeff;
    return w;
}

// The samples of w that stream s's output window (lwb_stream_set_window) lets through: w.skip and w.written.
static void clip_to_window(const lwb_stream *s, ChainWalk *w)
{
    window_clip(s->skip_left, s->limit_left, w->n_samples, &w->skip, &w->written);
}

static void set_chain_result(lwb_chain *c, const ChainWalk &w)
{
    c->status = w.status;
    c->packets_done = w.done;
    c->n_samples = (uint32_t)w.written;
}

// The stream states and output windows the walks of a batch leave, committed once the batch's work is queued.
static void commit_stream_states(const lwb_chain *chains, const std::vector<ChainWalk> &walks)
{
    for (size_t i = 0; i < walks.size(); i++) {
        lwb_stream *s = chains[i].stream;
        if (walks[i].done || walks[i].clear_after) set_stream_state(s, walks[i].end_has, walks[i].end_plen);
        s->skip_left -= walks[i].skip;
        if (s->limit_left != ~0ull) s->limit_left -= walks[i].written;
    }
}

// The three mode bytes (mode, previous and next window flag) of packet k of chain c, as the chain kernel reads them.
static void write_mode_bytes(const lwb_chain *c, uint32_t k, uint8_t *out)
{
    out[0] = c->mode_numbers[k];
    out[1] = c->prev_window_flags ? c->prev_window_flags[k] : 1;
    out[2] = c->next_window_flags ? c->next_window_flags[k] : 1;
}

// Cuts `whole`, the run of one channel (a LongRun or a ShortRun: in, out, state, in_stride, n_packets, has_prev), into
// `cuts` pieces w[0, cuts), for when there are too few runs to fill the machine.  Every piece after the first
// re-transforms the packet before its first one as a primer (its right half is all the piece needs), which keeps the
// pieces independent at the cost of one extra transform per cut.  Packet 0 of the run emits first_emit samples, every
// later one n2, of esz bytes each.  Only the last piece stores the state.
template <typename Run>
static void cut_run(const Run &whole, size_t cuts, size_t first_emit, size_t n2, size_t esz, Run *w)
{
    const size_t P = whole.n_packets;
    for (size_t k = 0; k < cuts; k++) {
        const size_t p0 = P * k / cuts, p1 = P * (k + 1) / cuts;   // this piece emits packets [p0, p1)
        Run &r = w[k];
        std::memset(&r, 0, sizeof(r));
        r.in_stride = whole.in_stride;
        r.state = whole.state;
        r.write_state = (k + 1 == cuts);
        if (k == 0) {
            r.in = whole.in;
            r.out = whole.out;
            r.n_packets = (uint32_t)(p1 - p0);
            r.has_prev = whole.has_prev;
        } else {
            const size_t primer = p0 - 1;
            r.in = whole.in + primer * whole.in_stride;
            r.out = (char *)whole.out + (first_emit + primer * n2) * esz;          // behind the samples before packet p0
            r.n_packets = (uint32_t)(p1 - p0 + 1);
            r.has_prev = 0;
        }
    }
}

// The run of channel ch of n packets of chain c, blocks of n2-point halves, cut into `cuts` pieces w[0, cuts): its
// coefficients start at `in` (the packets' first one; channels n2 apart, packets C * n2 apart), its PCM at `pcm` (the
// chain's sample of its first packet; planes out_stride apart, esz bytes per sample).  has: a state enters it;
// first_emit: the samples its first packet emits.
template <typename Run>
static void channel_run(const lwb_chain *c, unsigned ch, size_t n2, const float *in, char *pcm, size_t esz, uint32_t n, bool has,
                        size_t first_emit, size_t cuts, Run *w)
{
    const lwb_stream *s = c->stream;
    const lwb_setup *su = s->setup;
    const unsigned C = su->channels;
    cut_run(Run{in + (size_t)ch * n2, pcm + (c->out_offset + (size_t)ch * c->out_stride) * esz, s->d_state + (size_t)ch * state_stride(su),
                (uint32_t)(C * n2), n, has},
            cuts, first_emit, n2, esz, w);
}

// Static deals (run r -> warp r mod W: k_long_s, k_mid, k_short, k_short_g) finish with their most loaded warp: order the
// runs so that the W columns carry equal packet counts -- longest first, dealt boustrophedon (row 0 left to right, row 1
// right to left, ...).  With random run lengths an unordered deal leaves the slowest of 1184 warps a third above the mean.
// W: the warps of the launch of n runs, `warps` per CTA.
template <typename Run>
static void balance_static_deal(Run *runs, size_t n, int warps, int sm_count)
{
    const size_t W = (size_t)static_deal_grid(n, warps, sm_count) * warps;
    if (n <= W || W < 2) return;
    uint32_t maxp = 0;
    for (size_t i = 0; i < n; i++) maxp = std::max(maxp, runs[i].n_packets);
    std::vector<size_t> start(maxp + 2, 0);
    for (size_t i = 0; i < n; i++) start[maxp - runs[i].n_packets + 1]++;          // counting sort, descending
    for (size_t k = 1; k < start.size(); k++) start[k] += start[k - 1];
    std::vector<Run> tmp(n);
    const size_t full_rows = n / W;
    for (size_t i = 0; i < n; i++) {
        const size_t k = start[maxp - runs[i].n_packets]++;
        const size_t row = k / W, col = k % W;
        tmp[(row & 1) && row < full_rows ? row * W + (W - 1 - col) : k] = runs[i];
    }
    std::memcpy(runs, tmp.data(), n * sizeof(Run));
}

// Up to G runs of one length that a warp transforms in lockstep (k_mid, k_short_g); the deal above moves it as a unit.
template <typename Run, int G>
struct RunGroup { Run r[G]; uint32_t n_packets; };

// Cuts `runs` into groups of g <= G runs of equal length: longest first, in their order within a length.  The last group
// of a length is filled up with pad(its first run), a dummy of the kernel's own kind.  Sorts `runs`.
template <int G, typename Run, typename Pad>
static std::vector<RunGroup<Run, G>> group_runs(std::vector<Run> &runs, size_t g, Pad &&pad)
{
    std::stable_sort(runs.begin(), runs.end(), [](const Run &a, const Run &b) { return a.n_packets > b.n_packets; });
    std::vector<RunGroup<Run, G>> groups;
    for (size_t i = 0; i < runs.size();) {
        RunGroup<Run, G> &gr = groups.emplace_back();
        std::memset(&gr, 0, sizeof(gr));
        gr.n_packets = runs[i].n_packets;
        for (size_t k = 0; k < g; k++) gr.r[k] = i < runs.size() && runs[i].n_packets == gr.n_packets ? runs[i++] : pad(gr.r[0]);
    }
    return groups;
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

// The curves of the LWB_FLOOR_ZERO rows of n_pk packets with C channels into `curves` (addressed like the coefficient
// arena of the packets' coeff_off).
static int launch_floor0_curves(lwb_ctx *ctx, const DevPacket *d_pk, size_t n_pk, unsigned C, const uint8_t *kinds, const uint32_t *ys,
                                float *curves)
{
    const size_t rows = n_pk * C;
    if (!rows) return LWB_OK;
    return launch(ctx, LWB_KERNEL_FLOOR0_CURVES, k_floor0_curves, dim3((unsigned)((rows + kF0Rows - 1) / kF0Rows)), dim3(kF0Threads), 0, d_pk,
                  (uint32_t)rows, (int)C, kinds, ys, curves);
}

// n2max: the largest n/2 among the packets (sizes the per-row bin -> segment index).  floor0: the packets may have
// LWB_FLOOR_ZERO rows -- their curves are computed first, into ctx->floor0 at the offsets `spec` has in ctx->spec; without
// it (or without floor1_y) such rows act as LWB_FLOOR_UNUSED.
static int launch_prologue(lwb_ctx *ctx, const DevPacket *d_pk, size_t n_pk, unsigned C, bool fast, size_t smem_old, int n2max,
                           const float *res, const float *dense, const uint8_t *kinds, const uint32_t *ys, float *spec, VqView vq = VqView(),
                           bool floor0 = false)
{
    if (!n_pk) return LWB_OK;
    const int words = std::max(1, (n2max + 31) >> 5);
    if (vq.runs && (!fast || (size_t)C * n2max > kVqMaxElems))
        return fail(ctx, LWB_ERR_INVALID, "VQ entry needs <= 8 channels, aligned arenas and channels * n/2 <= 12288");
    int rc;
    float *zero = nullptr;
    if (floor0 && ys) {
        if ((rc = ensure(ctx, ctx->floor0, ctx->spec.cap))) return rc;
        zero = (float *)ctx->floor0.p + (spec - (float *)ctx->spec.p);
        if ((rc = launch_floor0_curves(ctx, d_pk, n_pk, C, kinds, ys, zero))) return rc;
    }
    if (!fast)
        return launch(ctx, LWB_KERNEL_PROLOGUE, k_prologue, dim3((unsigned)n_pk), dim3(kPrologueThreads), smem_old, d_pk, res, dense, kinds, ys, spec,
                      (const float *)zero);
    // per (packet, channel) row (ctx scratch): the packed flagged segments of its floor curve, the bin -> segment
    // index (bitmap + prefix counts) and the segment count
    const size_t rows = n_pk * C, tab_bytes = rows * kSegStride * sizeof(uint4), ix_bytes = rows * seg_index_stride(words);
    if ((rc = ensure(ctx, ctx->segtab, tab_bytes + ix_bytes + rows + 64))) return rc;
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
                      (uint32_t)n_pk, res, dense, (const float *)zero, kinds, (const uint4 *)tab, (const uint8_t *)cnt, (const unsigned char *)ix, words, spec, vd);
    return launch(ctx, LWB_KERNEL_PROLOGUE_FUSED, k_prologue_fused<false>, dim3((unsigned)grid), dim3(kPfThreads), prologue_fused_smem((int)C, words), d_pk, (uint32_t)n_pk, res, dense,
                  (const float *)zero, kinds, (const uint4 *)tab, (const uint8_t *)cnt, (const unsigned char *)ix, words, spec, vd);
}
static int launch_prologue(lwb_ctx *ctx, const DevPacket *d_pk, const DevPacket *h_pk, size_t n_pk, unsigned C, size_t smem_old,
                           const float *res, const float *dense, const uint8_t *kinds, const uint32_t *ys, float *spec, VqView vq, bool floor0)
{
    int n2max = 32;
    for (size_t i = 0; i < n_pk; i++) n2max = std::max(n2max, h_pk[i].n >> 1);
    return launch_prologue(ctx, d_pk, n_pk, C, prologue_is_fast(h_pk, n_pk, C, res, dense, spec), smem_old, n2max, res, dense, kinds, ys, spec, vq,
                           floor0);
}

// Host-side look at the floor kinds of the `done` packets chain c decodes (one row per (packet, channel)).  Device-resident
// floor arrays (io->floor_memory == LWB_MEM_DEVICE) cannot be looked at: they are trusted, and the batch is assumed
// to carry dense (floor-0) curves exactly when the caller passed a dense_floor arena, and floor-0 records exactly when
// the chain's setup has floor-0 descriptions.
static int scan_floor_kinds(lwb_ctx *ctx, const lwb_batch_io *io, const lwb_chain *c, uint32_t done, bool *need_dense, bool *need_floor0)
{
    const lwb_setup *su = c->stream->setup;
    if (io->floor_memory == LWB_MEM_DEVICE) {
        if (io->dense_floor) *need_dense = true;
        if (!su->floor0.empty()) *need_floor0 = true;
        return LWB_OK;
    }
    const unsigned C = su->channels;
    for (uint32_t k = 0; k < done; k++) {
        const uint8_t *kinds = io->floor_kind + (c->packet_index + k) * C;
        for (unsigned ch = 0; ch < C; ch++) {
            const uint8_t kd = kinds[ch];
            if (kd > LWB_FLOOR_ZERO) return fail(ctx, LWB_ERR_INVALID, "floor_kind out of range");
            if ((kd == LWB_FLOOR_ONE || kd == LWB_FLOOR_ZERO) && !io->floor1_y) return fail(ctx, LWB_ERR_INVALID, "floor1_y missing");
            if (kd == LWB_FLOOR_DENSE) *need_dense = true;
            if (kd != LWB_FLOOR_ZERO) continue;
            const DevMapping &mp = su->mappings[su->host.mode_mapping[c->mode_numbers[k]]];
            if (!su->floor0_described(mp.floor_of_channel[ch]))
                return fail(ctx, LWB_ERR_INVALID, "floor_kind out of range: LWB_FLOOR_ZERO on a floor without a floor-0 description");
            *need_floor0 = true;
        }
    }
    return LWB_OK;
}

// Host VQ offsets (LWB_ENTRY_VQ) bound the records of packet rows [r_lo, r_hi), which floor_views stages: they must not
// decrease across them.  Device arrays cannot be looked at.
static int check_vq_offsets(lwb_ctx *ctx, const lwb_batch_io *io, uint64_t r_lo, uint64_t r_hi)
{
    if (io->entry != LWB_ENTRY_VQ || io->floor_memory == LWB_MEM_DEVICE || r_hi <= r_lo) return LWB_OK;
    if (io->vq_run_offsets[r_hi] < io->vq_run_offsets[r_lo] || io->vq_entry_offsets[r_hi] < io->vq_entry_offsets[r_lo])
        return fail(ctx, LWB_ERR_INVALID, "vq offsets must be non-decreasing");
    return LWB_OK;
}

// The floor and VQ arrays (LWB_ENTRY_VQ) of packet rows [r_lo, r_hi) of a batch with C channels as the device sees
// them, biased so that ABSOLUTE rows and offsets address them.  Host arrays get room in the kinds / ys / vqoff / vqrec
// arenas of `set` (grown behind `in_use`, see ensure()), which upload_floor_rows fills; device arrays are used in place.
// The caller has checked the VQ offsets (check_vq_offsets).
struct FloorViews {
    const uint8_t *kinds = nullptr;
    const uint32_t *ys = nullptr;
    VqView vq;
};

static int floor_views(lwb_ctx *ctx, const lwb_batch_io *io, ArenaSet &set, cudaEvent_t in_use, uint64_t r_lo, uint64_t r_hi,
                       unsigned C, FloorViews *v)
{
    *v = FloorViews();
    if (io->entry == LWB_ENTRY_SPECTRUM) return LWB_OK;
    const bool vq = io->entry == LWB_ENTRY_VQ;
    if (io->floor_memory == LWB_MEM_DEVICE) {
        v->kinds = io->floor_kind;
        v->ys = io->floor1_y;
        if (vq) v->vq = VqView{io->vq_runs, io->vq_run_offsets, io->vq_entries, io->vq_entry_offsets};
        return LWB_OK;
    }
    if (r_hi <= r_lo) return LWB_OK;
    int rc;
    const size_t rows = (size_t)(r_hi - r_lo) * C;
    if ((rc = ensure(ctx, set.kinds, rows, in_use))) return rc;
    v->kinds = (const uint8_t *)set.kinds.p - r_lo * C;
    if (io->floor1_y) {
        if ((rc = ensure(ctx, set.ys, rows * LWB_MAX_POSTS * sizeof(uint32_t), in_use))) return rc;
        v->ys = (const uint32_t *)set.ys.p - r_lo * C * LWB_MAX_POSTS;
    }
    if (!vq) return LWB_OK;
    const uint64_t o_lo = io->vq_run_offsets[r_lo], o_hi = io->vq_run_offsets[r_hi];
    const uint64_t e_lo = io->vq_entry_offsets[r_lo], e_hi = io->vq_entry_offsets[r_hi];
    const size_t b_off = ((size_t)(r_hi - r_lo) + 1) * sizeof(uint64_t), b_run = std::max<size_t>((size_t)(o_hi - o_lo), 1) * sizeof(lwb_vq_run);
    if ((rc = ensure(ctx, set.vqoff, 2 * b_off, in_use)) ||
        (rc = ensure(ctx, set.vqrec, b_run + std::max<size_t>((size_t)(e_hi - e_lo), 1) * sizeof(uint16_t) + 16, in_use)))
        return rc;
    v->vq.run_off = (const uint64_t *)set.vqoff.p - r_lo;
    v->vq.ent_off = (const uint64_t *)((char *)set.vqoff.p + b_off) - r_lo;
    v->vq.runs = (const lwb_vq_run *)set.vqrec.p - o_lo;
    v->vq.entries = (const uint16_t *)((char *)set.vqrec.p + b_run) - e_lo;
    return LWB_OK;
}

// H2D of the host floor and VQ arrays of rows [a, b) into views v, on `sm`.
static int upload_floor_rows(lwb_ctx *ctx, const lwb_batch_io *io, uint64_t a, uint64_t b, unsigned C, const FloorViews &v, cudaStream_t sm)
{
    if (io->entry == LWB_ENTRY_SPECTRUM || io->floor_memory == LWB_MEM_DEVICE || b <= a) return LWB_OK;
    const size_t rows = (size_t)(b - a) * C;
    CU(ctx, cudaMemcpyAsync(const_cast<uint8_t *>(v.kinds) + a * C, io->floor_kind + a * C, rows, cudaMemcpyHostToDevice, sm));
    if (io->floor1_y)
        CU(ctx, cudaMemcpyAsync(const_cast<uint32_t *>(v.ys) + a * C * LWB_MAX_POSTS, io->floor1_y + a * C * LWB_MAX_POSTS,
                                rows * LWB_MAX_POSTS * sizeof(uint32_t), cudaMemcpyHostToDevice, sm));
    if (io->entry != LWB_ENTRY_VQ) return LWB_OK;
    const uint64_t o_a = io->vq_run_offsets[a], o_b = io->vq_run_offsets[b], e_a = io->vq_entry_offsets[a], e_b = io->vq_entry_offsets[b];
    const size_t b_off = ((size_t)(b - a) + 1) * sizeof(uint64_t);
    CU(ctx, cudaMemcpyAsync(const_cast<uint64_t *>(v.vq.run_off) + a, io->vq_run_offsets + a, b_off, cudaMemcpyHostToDevice, sm));
    CU(ctx, cudaMemcpyAsync(const_cast<uint64_t *>(v.vq.ent_off) + a, io->vq_entry_offsets + a, b_off, cudaMemcpyHostToDevice, sm));
    if (o_b > o_a) CU(ctx, cudaMemcpyAsync(const_cast<lwb_vq_run *>(v.vq.runs) + o_a, io->vq_runs + o_a, (size_t)(o_b - o_a) * sizeof(lwb_vq_run), cudaMemcpyHostToDevice, sm));
    if (e_b > e_a) CU(ctx, cudaMemcpyAsync(const_cast<uint16_t *>(v.vq.entries) + e_a, io->vq_entries + e_a, (size_t)(e_b - e_a) * sizeof(uint16_t), cudaMemcpyHostToDevice, sm));
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// extent and host-memory pipeline of a batch
// ---------------------------------------------------------------------------------------------
// The ranges a batch, or a chunk of it, reads and writes: coefficient elements [c_lo, c_hi), PCM elements [o_lo, o_hi)
// and, for the residue entries, packet rows [r_lo, r_hi).
struct BatchExtent {
    uint64_t c_lo = ~0ull, c_hi = 0, o_lo = ~0ull, o_hi = 0, r_lo = ~0ull, r_hi = 0;
    bool need_dense = false;      // a decoded row has a dense floor
    bool need_floor0 = false;     // a decoded row may have a floor-0 record (LWB_FLOOR_ZERO)

    // The ranges of chain c, whose walk w decodes w.done packets and writes w.written samples per channel.
    void add(const lwb_batch_io *io, const lwb_chain *c, const ChainWalk &w)
    {
        if (!w.done) return;
        const unsigned C = c->stream->setup->out_channels();
        const bool planar = out_format_of(io->out_format).planar;
        c_lo = std::min(c_lo, c->coeff_offset);
        c_hi = std::max(c_hi, w.coeff_end);
        o_lo = std::min(o_lo, c->out_offset);
        o_hi = std::max(o_hi, c->out_offset + (planar ? (uint64_t)(C - 1) * c->out_stride + w.written : w.written * C));
        if (io->entry == LWB_ENTRY_SPECTRUM) return;
        r_lo = std::min(r_lo, c->packet_index);
        r_hi = std::max<uint64_t>(r_hi, c->packet_index + w.done);
    }
    bool empty() const { return c_hi <= c_lo; }
};

// A batch walked once, before a path is chosen (walk_batch, lwb_api.cu): every chain's walk and the batch's extent.
// The paths read it; queue_batch writes the chain results and stream states from it once a path has queued the batch.
// `clip` (place_clipped_chains, lwb_api.cu) is empty unless a chain's window clips it: it is then the chain array the
// paths decode, in which each clipped chain writes its full output to scratch; BatchArenas::download moves the written
// samples to their place in the caller's chains.
struct BatchWalk {
    const lwb_chain *chains = nullptr;      // the caller's
    std::vector<ChainWalk> walks;
    BatchExtent ext;
    std::vector<lwb_chain> clip;
};

// The extent of chains [i0, i1) of a walked batch: one chunk of a chunked host-memory batch.
static BatchExtent chunk_extent(const lwb_batch_io *io, const lwb_chain *chains, const BatchWalk &bw, size_t i0, size_t i1)
{
    BatchExtent e;
    for (size_t i = i0; i < i1; i++) e.add(io, &chains[i], bw.walks[i]);
    return e;
}

// Whether host bytes [lo, hi) * esz of `base` begin and end in page-locked memory (the runtime tells; pageable memory
// is "unregistered").
static bool page_locked(const void *base, uint64_t lo, uint64_t hi, size_t esz)
{
    if (hi <= lo) return true;
    for (const char *p : {(const char *)base + lo * esz, (const char *)base + hi * esz - 1}) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        if (a.type != cudaMemoryTypeHost) return false;
    }
    return true;
}

// A host-memory submit copies straight from and to the caller's arrays, after the call has returned: every range of
// them the batch touches must be page-locked.
static int check_page_locked(lwb_ctx *ctx, const lwb_batch_io *io, const BatchExtent &ext, unsigned C)
{
    const char *bad = nullptr;
    if (io->entry != LWB_ENTRY_VQ && !page_locked(io->coeffs, ext.c_lo, ext.c_hi, sizeof(float))) bad = "coeffs";
    else if (ext.need_dense && !page_locked(io->dense_floor, ext.c_lo, ext.c_hi, sizeof(float))) bad = "dense_floor";
    else if (!page_locked(io->pcm, ext.o_lo, ext.o_hi, out_format_of(io->out_format).esz)) bad = "pcm";
    else if (io->entry != LWB_ENTRY_SPECTRUM && io->floor_memory == LWB_MEM_HOST && ext.r_hi > ext.r_lo) {
        const uint64_t a = ext.r_lo * C, b = ext.r_hi * C;
        if (!page_locked(io->floor_kind, a, b, 1)) bad = "floor_kind";
        else if (io->floor1_y && !page_locked(io->floor1_y, a * LWB_MAX_POSTS, b * LWB_MAX_POSTS, sizeof(uint32_t))) bad = "floor1_y";
        else if (io->entry == LWB_ENTRY_VQ) {
            if (!page_locked(io->vq_run_offsets, ext.r_lo, ext.r_hi + 1, sizeof(uint64_t))) bad = "vq_run_offsets";
            else if (!page_locked(io->vq_entry_offsets, ext.r_lo, ext.r_hi + 1, sizeof(uint64_t))) bad = "vq_entry_offsets";
            else if (!page_locked(io->vq_runs, io->vq_run_offsets[ext.r_lo], io->vq_run_offsets[ext.r_hi], sizeof(lwb_vq_run))) bad = "vq_runs";
            else if (!page_locked(io->vq_entries, io->vq_entry_offsets[ext.r_lo], io->vq_entry_offsets[ext.r_hi], sizeof(uint16_t))) bad = "vq_entries";
        }
    }
    if (!bad) return LWB_OK;
    return fail(ctx, LWB_ERR_INVALID, (std::string("host-memory submit: ") + bad +
                                       " is not page-locked (lwb_host_alloc, cudaHostAlloc or cudaHostRegister)").c_str());
}

// D2H of the PCM that chains [i0, i1), walked as walks[i0, i1), wrote, from the staging buffer `stage`, which holds
// arena element `obase` at its start.  Only the write set is copied (pcm_copy_plan.h): the gaps between planes and
// between chains are the caller's memory, and the kernels never wrote them in the staging buffer.
static int copy_pcm_to_host(lwb_ctx *ctx, const lwb_batch_io *io, const lwb_chain *chains, const ChainWalk *walks, size_t i0, size_t i1,
                            const void *stage, uint64_t obase, cudaStream_t st)
{
    const size_t esz = out_format_of(io->out_format).esz;
    const bool planar = out_format_of(io->out_format).planar;
    ctx->pcm_spans.clear();
    for (size_t i = i0; i < i1; i++) {
        const lwb_chain *c = &chains[i];
        pcm_chain_spans(planar, c->stream->setup->out_channels(), c->out_offset, c->out_stride, walks[i].written, ctx->pcm_spans);
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

// The arenas of a batch as its kernels address them: coefficients, dense floors and PCM by absolute element offset,
// floor and VQ arrays by absolute packet row (FloorViews).  A host-memory batch is staged in the next of the context's
// host sets, chunk by chunk: upload(k) brings chunk k's inputs, download(k) takes its PCM home behind its kernels.  Its
// uploads wait on the GPU for the batch that used the set before (ArenaSet::done) and nothing else.  With the copy
// streams (copy_in / copy_out, ordered by ev_in[k] / ev_done[k]) the copies of one chunk overlap the kernels of
// another; otherwise everything runs on the compute stream.  A device-memory batch uses the caller's arenas in place.
static int run_steps(lwb_ctx *ctx, const StepArgs &a, const std::vector<Step> &steps);

struct BatchArenas {
    const float *coeffs = nullptr, *dense = nullptr;
    char *pcm = nullptr;
    FloorViews fl;
    lwb_ctx *ctx = nullptr;
    const lwb_batch_io *io = nullptr;
    ArenaSet *set = nullptr;
    bool host = false;
    unsigned C = 0;
    uint64_t c_lo = 0, o_lo = 0;
    cudaStream_t up = nullptr, down = nullptr;

    int open(lwb_ctx *ctx_, const lwb_batch_io *io_, const BatchExtent &ext, unsigned C_, bool copy_streams)
    {
        ctx = ctx_;
        io = io_;
        C = C_;
        c_lo = ext.c_lo;
        o_lo = ext.o_lo;
        host = io->memory == LWB_MEM_HOST;
        const bool vq = io->entry == LWB_ENTRY_VQ;
        up = host && copy_streams ? ctx->copy_in : ctx->stream;
        down = host && copy_streams ? ctx->copy_out : ctx->stream;
        int rc;
        cudaEvent_t in_use = nullptr;
        if (host) {
            set = &ctx->host_sets[ctx->host_next];
            ctx->host_next = (ctx->host_next + 1) % kHostSets;
            in_use = set->done;
            const size_t esz = out_format_of(io->out_format).esz, bytes = (size_t)(ext.c_hi - ext.c_lo) * sizeof(float);
            if (ext.o_hi > ext.o_lo && (rc = ensure(ctx, set->pcm, (size_t)(ext.o_hi - ext.o_lo) * esz, in_use))) return rc;
            if (!vq && (rc = ensure(ctx, set->coeffs, bytes, in_use))) return rc;
            if (ext.need_dense && (rc = ensure(ctx, set->dense, bytes, in_use))) return rc;
            coeffs = vq ? nullptr : (const float *)set->coeffs.p - c_lo;
            dense = ext.need_dense ? (const float *)set->dense.p - c_lo : nullptr;
            pcm = (char *)set->pcm.p - o_lo * esz;
        } else {
            set = &ctx->ordered;
            coeffs = vq ? nullptr : io->coeffs;
            dense = io->dense_floor;
            pcm = (char *)io->pcm;
        }
        if ((rc = floor_views(ctx, io, *set, in_use, ext.r_lo, ext.r_hi, C, &fl))) return rc;
        if (host) CU(ctx, cudaStreamWaitEvent(up, set->done, 0));
        return LWB_OK;
    }
    int upload(size_t k, const BatchExtent &ck)
    {
        int rc;
        if (host) {
            const size_t bytes = (size_t)(ck.c_hi - ck.c_lo) * sizeof(float);
            if (coeffs) CU(ctx, cudaMemcpyAsync(const_cast<float *>(coeffs) + ck.c_lo, io->coeffs + ck.c_lo, bytes, cudaMemcpyHostToDevice, up));
            if (dense) CU(ctx, cudaMemcpyAsync(const_cast<float *>(dense) + ck.c_lo, io->dense_floor + ck.c_lo, bytes, cudaMemcpyHostToDevice, up));
        }
        if ((rc = upload_floor_rows(ctx, io, ck.r_lo, ck.r_hi, C, fl, up))) return rc;
        if (up == ctx->stream) return LWB_OK;
        CU(ctx, cudaEventRecord(ctx->ev_in[k], up));
        CU(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[k], 0));
        return LWB_OK;
    }
    // Chains [i0, i1) of the batch make up chunk k, whose kernels are queued: the written samples of its clipped chains
    // go to their place, then a host-memory batch's PCM goes home.
    int download(size_t k, const BatchWalk &bw, size_t i0, size_t i1, const BatchExtent &ck)
    {
        int rc;
        if (!bw.clip.empty() && (rc = move_clipped(bw, i0, i1))) return rc;
        if (!host || ck.o_hi <= ck.o_lo) return LWB_OK;
        if (down != ctx->stream) {
            CU(ctx, cudaEventRecord(ctx->ev_done[k], ctx->stream));
            CU(ctx, cudaStreamWaitEvent(down, ctx->ev_done[k], 0));
        }
        return copy_pcm_to_host(ctx, io, bw.chains, bw.walks.data(), i0, i1, set->pcm.p, o_lo, down);
    }
    // One k_row_copy launch on the compute stream: per clipped chain of [i0, i1) with written samples, per plane (or the
    // one interleaved range), samples [skip, skip + written) of its full output (bw.clip) to the caller's place.
    int move_clipped(const BatchWalk &bw, size_t i0, size_t i1)
    {
        const OutFormat of = out_format_of(io->out_format);
        size_t n = 0;
        for (size_t i = i0; i < i1; i++)
            if (bw.walks[i].clipped() && bw.walks[i].written) n += of.planar ? bw.chains[i].stream->setup->out_channels() : 1;
        if (!n) return LWB_OK;
        Staging *st;
        int rc;
        if ((rc = acquire_staging(ctx, n * sizeof(RowCopy), &st)) || (rc = ensure(ctx, ctx->state_rows, n * sizeof(RowCopy)))) return rc;
        RowCopy *h = (RowCopy *)st->h, *w = h;
        for (size_t i = i0; i < i1; i++) {
            const ChainWalk &cw = bw.walks[i];
            if (!cw.clipped() || !cw.written) continue;
            const lwb_chain &c = bw.chains[i], &full = bw.clip[i];
            const uint64_t K = c.stream->setup->out_channels();
            if (!of.planar) {
                *w++ = RowCopy{pcm + (full.out_offset + cw.skip * K) * of.esz, pcm + c.out_offset * of.esz, cw.written * K * of.esz};
                continue;
            }
            for (uint64_t k = 0; k < K; k++)
                *w++ = RowCopy{pcm + (full.out_offset + k * full.out_stride + cw.skip) * of.esz, pcm + (c.out_offset + k * c.out_stride) * of.esz,
                               cw.written * of.esz};
        }
        if ((rc = upload_staging(ctx, st, h, ctx->state_rows.p, n * sizeof(RowCopy), ctx->stream))) return rc;
        return run_steps(ctx, StepArgs(), std::vector<Step>(1, Step{LWB_KERNEL_ROW_COPY, ctx->state_rows.p, n, nullptr}));
    }
    // The batch is queued: a host-memory batch records its ticket, which also releases its set to the next user.
    int finish()
    {
        finished = true;
        return host ? issue_ticket(ctx, set) : LWB_OK;
    }
    // A host-memory batch that failed after open() still releases its set behind whatever it had queued, so that the
    // set's next user waits for copies and kernels that may still read it.  (Failures here are dropped: the batch
    // already reports the first one.)
    ~BatchArenas()
    {
        if (!host || !set || finished) return;
        cudaEventRecord(ctx->ev_done[64], ctx->copy_in);
        cudaStreamWaitEvent(ctx->stream, ctx->ev_done[64], 0);
        cudaEventRecord(ctx->ev_done[64], ctx->stream);
        cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[64], 0);
        cudaEventRecord(set->done, ctx->copy_out);
        cudaGetLastError();
    }
    bool finished = false;
};

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

// The arenas the front stages read and write, biased by fs.c_lo (== the c_lo of the batch's arenas ar): residues and
// dense floors as ar holds them (the caller's in device memory, their staged copies in host memory), and ctx->spec.
struct FrontArenas { const float *res, *dense; float *spec; };
static FrontArenas front_arenas(lwb_ctx *ctx, const BatchArenas &ar, const FrontStages &fs)
{
    return FrontArenas{ar.coeffs, fs.dense ? ar.dense : nullptr, (float *)ctx->spec.p - fs.c_lo};
}

// Whether the two-kernel form takes fs's packets (host copy h_pk of its list).
static bool front_stages_fast(lwb_ctx *ctx, const BatchArenas &ar, const FrontStages &fs, const DevPacket *h_pk)
{
    const FrontArenas a = front_arenas(ctx, ar, fs);
    return prologue_is_fast(h_pk, fs.n, fs.C, a.res, a.dense, a.spec);
}

// The front stages of n packets with C channels, none larger than n1max, over the arenas of `ext`; the packet list
// (pk, fast) is the caller's.
static FrontStages front_stages_of(const BatchExtent &ext, unsigned C, int n1max, size_t n)
{
    FrontStages fs;
    fs.n = n;
    fs.C = C;
    fs.smem_old = prologue_smem((int)C, __builtin_ctz((unsigned)n1max));
    fs.n2max = n1max >> 1;
    fs.c_lo = ext.c_lo;
    fs.r_lo = ext.r_lo;
    fs.r_hi = ext.r_hi;
    fs.dense = ext.need_dense;
    fs.floor0 = ext.need_floor0;
    return fs;
}

// Writes the packet list of every packet of chains [0, n_chains) into ring staging and uploads it, on the compute
// stream, to `off` bytes into `db`: fs->pk and fs->fast.
static int stage_front_packets(lwb_ctx *ctx, const BatchArenas &ar, const lwb_chain *chains, size_t n_chains, DevBuf &db, size_t off,
                               FrontStages *fs)
{
    const size_t bytes = fs->n * sizeof(DevPacket);
    Staging *st;
    int rc;
    if ((rc = acquire_staging(ctx, bytes, &st)) || (rc = ensure(ctx, db, off + bytes))) return rc;
    DevPacket *hp = (DevPacket *)st->h, *w = hp;
    for (size_t i = 0; i < n_chains; i++) {
        write_front_packets(&chains[i], 0, chains[i].n_packets, chains[i].coeff_offset, w);
        w += chains[i].n_packets;
    }
    fs->pk = (const DevPacket *)((char *)db.p + off);
    fs->fast = front_stages_fast(ctx, ar, *fs, hp);
    return upload_staging(ctx, st, hp, (char *)db.p + off, bytes, ctx->stream);
}

// Packets [k0, k0 + n) of fs on the floor / VQ views of ar, which the caller has staged.
static int front_stages_launch(lwb_ctx *ctx, const BatchArenas &ar, const FrontStages &fs, size_t k0, size_t n)
{
    const FrontArenas a = front_arenas(ctx, ar, fs);
    return launch_prologue(ctx, fs.pk + k0, n, fs.C, fs.fast, fs.smem_old, fs.n2max, a.res, a.dense, ar.fl.kinds, ar.fl.ys, a.spec, ar.fl.vq,
                           fs.floor0);
}

// A device-memory batch's front stages alone: stages the floor and VQ arrays of fs's packet rows on the compute stream
// (host arrays are uploaded, device arrays read in place) and launches the front stages over every packet of fs.
static int front_stages_run(lwb_ctx *ctx, const lwb_batch_io *io, const FrontStages &fs)
{
    BatchExtent ext;
    ext.c_lo = fs.c_lo;
    ext.r_lo = fs.r_lo;
    ext.r_hi = fs.r_hi;
    ext.need_dense = fs.dense;
    BatchArenas ar;
    int rc;
    if ((rc = check_vq_offsets(ctx, io, fs.r_lo, fs.r_hi)) || (rc = ar.open(ctx, io, ext, fs.C, false)) || (rc = ar.upload(0, ext))) return rc;
    return front_stages_launch(ctx, ar, fs, 0, fs.n);
}

// ---------------------------------------------------------------------------------------------
// the launches of the fused paths and the chain-kernel path (Step)
// ---------------------------------------------------------------------------------------------
// k_chain for the batch's entry, output format, mix and warps per chain
static int launch_chain(lwb_ctx *ctx, const StepArgs &a, uint32_t n_chains, const ChainDesc *d)
{
    auto entry = [&](auto go) {
        switch (a.entry) {
        case LWB_ENTRY_VQ: return go(std::integral_constant<int, LWB_ENTRY_VQ>());
        case LWB_ENTRY_RESIDUE: return go(std::integral_constant<int, LWB_ENTRY_RESIDUE>());
        default: return go(std::integral_constant<int, LWB_ENTRY_SPECTRUM>());
        }
    };
    return entry([&](auto e) {
        return with_out_format(a.out_format, [&](auto f) {
            constexpr int ENTRY = decltype(e)::value, F = decltype(f)::value;
            auto go = [&](auto wide, auto mix) {         // wide: more than one warp per chain
                constexpr bool WIDE = decltype(wide)::value, MIX = decltype(mix)::value;
                cudaFuncSetAttribute(k_chain<F, ENTRY, WIDE, MIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)a.chain.smem);
                return launch(ctx, LWB_KERNEL_CHAIN, k_chain<F, ENTRY, WIDE, MIX>, dim3(n_chains), dim3(a.chain.warps * 32), a.chain.smem, d,
                              a.bytes, a.coeffs, a.dense, a.kinds, a.ys, a.pcm, a.chain.n1max, a.chain.wpc, WIDE ? 1 : a.chain.np, a.zero, a.vq);
            };
            const std::true_type yes;
            const std::false_type no;
            if (a.chain.wpc == 1) return a.mix ? go(no, yes) : go(no, no);
            return a.mix ? go(yes, yes) : go(yes, no);
        });
    });
}

__global__ void __launch_bounds__(kRowCopyThreads) k_row_copy(const RowCopy *__restrict__ rc);   // path_chain.cuh

// Launches `steps` in order on the compute stream.  Only k_long draws a ticket.
static int run_steps(lwb_ctx *ctx, const StepArgs &a, const std::vector<Step> &steps)
{
    cudaStream_t sm = ctx->stream;
    const SampleKind kind = out_format_of(a.out_format).kind;
    for (const Step &s : steps) {
        int rc;
        unsigned int *ticket;
        const uint32_t n = (uint32_t)s.n;
        switch (s.kernel) {
        case LWB_KERNEL_ROW_COPY:
            rc = launch(ctx, LWB_KERNEL_ROW_COPY, k_row_copy, dim3(n), dim3(kRowCopyThreads), 0, (const RowCopy *)s.desc);
            break;
        case LWB_KERNEL_LONG:
            if ((rc = next_ticket(ctx, &ticket))) return rc;
            rc = launched(ctx, LWB_KERNEL_LONG, long_launch(sm, (const LongRun *)s.desc, n, s.pack, ticket, ctx->sm_count, kind, a.w_short, a.ls),
                          "long kernel launch");
            break;
        case LWB_KERNEL_LONG_S:         // one pass over many short runs: the static deal with its deeper lookahead
            rc = launched(ctx, LWB_KERNEL_LONG_S, long_launch_static(sm, (const LongRun *)s.desc, n, s.pack, ctx->sm_count, kind, a.w_short, a.ls),
                          "long kernel launch");
            break;
        case LWB_KERNEL_MID:
            rc = launched(ctx, LWB_KERNEL_MID, mid_launch(sm, (const LongRun *)s.desc, n, s.pack, ctx->sm_count, kind, a.mid_kb), "mid kernel launch");
            break;
        case LWB_KERNEL_SHORT:
            rc = launched(ctx, LWB_KERNEL_SHORT, short_launch(sm, (const ShortRun *)s.desc, n, s.pack, ctx->sm_count, kind), "short kernel launch");
            break;
        case LWB_KERNEL_SHORT_G:        // bursts: eight short runs of equal length per warp
            rc = launched(ctx, LWB_KERNEL_SHORT_G, short_launch_groups(sm, (const ShortRun *)s.desc, n, s.pack, ctx->sm_count, kind),
                          "short burst kernel launch");
            break;
        case LWB_KERNEL_CHAIN:
            rc = launch_chain(ctx, a, n, (const ChainDesc *)s.desc);
            break;
        default:
            return fail(ctx, LWB_ERR_INVALID, "internal: no step for this kernel");
        }
        if (rc) return rc;
    }
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// four-kernel path (kernels_generic.cuh): the last batch path, which takes every batch that reaches it
// ---------------------------------------------------------------------------------------------
struct PlanPacket {
    Geom g;
    uint32_t plen;          // 0: no previous half -> 0 samples out
    uint64_t coeff_off;     // absolute element offset
    uint64_t sample_pos;    // samples (per channel) produced by the chain before this packet
};

struct PlanChain {
    const lwb_chain *c;
    std::vector<PlanPacket> pk;
};

// dynamic shared memory k_prologue needs for the chains of a batch (curve bytes of the largest block)
static size_t prologue_smem_of(const std::vector<PlanChain> &plan)
{
    size_t m = 0;
    for (const PlanChain &pc : plan)
        if (pc.c && pc.c->stream) m = std::max(m, prologue_smem(pc.c->stream->setup->channels, pc.c->stream->setup->bs1));
    return m;
}

// Rounds of packets bounded by the IMDCT scratch.  Each round stages its descriptors in the next slot of the staging
// ring; ctx->desc, ctx->x and ctx->spec are reused from round to round in compute-stream order.  The descriptors
// address a host-memory batch's staging from its start (element c_lo / o_lo), a device-memory batch's arenas from
// element 0.  ext_floor0: the batch may have LWB_FLOOR_ZERO rows (BatchExtent::need_floor0).
static int run_generic(lwb_ctx *ctx, std::vector<PlanChain> &plan, const lwb_batch_io *io, const BatchArenas &ar, bool ext_floor0)
{
    size_t maxp = 0;
    for (auto &pc : plan) maxp = std::max(maxp, pc.pk.size());
    if (maxp == 0) return LWB_OK;
    const uint64_t coeff_base = ar.host ? ar.c_lo : 0, pcm_base = ar.host ? ar.o_lo : 0;
    const float *coeffs = ar.coeffs ? ar.coeffs + coeff_base : nullptr, *dense = ar.dense ? ar.dense + coeff_base : nullptr;
    void *pcm = ar.pcm + pcm_base * out_format_of(io->out_format).esz;
    // x elements of one "packet column" (packet i of every chain), to size the rounds
    std::vector<uint32_t> start(plan.size(), 0);
    const bool planar = out_format_of(io->out_format).planar;
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
        Staging *st;
        if ((rc = acquire_staging(ctx, n_desc * sizeof(DevPacket), &st)) || (rc = ensure(ctx, ctx->desc, n_desc * sizeof(DevPacket))) ||
            (rc = ensure(ctx, ctx->x, x_elems * sizeof(float))))
            return rc;
        DevPacket *hp = (DevPacket *)st->h;
        size_t di = 0, xo = 0;
        unsigned maxc = 1, maxn = 64, maxk = 1;
        bool mix = false;
        for (size_t ci = 0; ci < plan.size(); ci++) {
            PlanChain &pc = plan[ci];
            const lwb_stream *s = pc.c->stream;
            const lwb_setup *su = s->setup;
            const unsigned C = su->channels, K = su->out_channels();
            if (take[ci]) {
                maxk = std::max(maxk, K);
                mix |= su->host.n_out != 0;
            }
            for (uint32_t k = 0; k < take[ci]; k++) {
                const PlanPacket &pp = pc.pk[start[ci] + k];
                DevPacket &d = hp[di];
                std::memset(&d, 0, sizeof(d));
                d.setup = su->d_setup;
                d.state = s->d_state;
                d.coeff_off = pp.coeff_off - coeff_base;
                d.x_off = xo;
                d.out_stride = pc.c->out_stride;
                d.out_off = pc.c->out_offset - pcm_base + (planar ? pp.sample_pos : pp.sample_pos * K);
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
        if ((rc = upload_staging(ctx, st, hp, ctx->desc.p, n_desc * sizeof(DevPacket), ctx->stream))) return rc;
        const DevPacket *dp = (const DevPacket *)ctx->desc.p;
        const float *spec = coeffs;
        if (io->entry != LWB_ENTRY_SPECTRUM) {
            if ((rc = ensure(ctx, ctx->spec, spec_hi * sizeof(float)))) return rc;
            if ((rc = launch_prologue(ctx, dp, hp, n_desc, maxc, prologue_smem_of(plan), coeffs, dense, ar.fl.kinds, ar.fl.ys,
                                      (float *)ctx->spec.p, ar.fl.vq, ext_floor0)))
                return rc;
            spec = (const float *)ctx->spec.p;
        }
        if ((rc = launch(ctx, LWB_KERNEL_IMDCT, k_imdct, dim3((unsigned)n_desc, maxc), dim3(kImdctThreads), maxn * sizeof(float), dp,
                         spec, (float *)ctx->x.p)))
            return rc;
        dim3 g2((unsigned)n_desc, maxc), b2(kOverlapThreads);
        rc = with_out_format(io->out_format, [&](auto f) {
            if (mix)        // grid.y: output channels
                return launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<decltype(f)::value, true>, dim3((unsigned)n_desc, maxk), b2, 0, dp,
                              (const float *)ctx->x.p, pcm);
            return launch(ctx, LWB_KERNEL_OVERLAP, k_overlap<decltype(f)::value>, g2, b2, 0, dp, (const float *)ctx->x.p, pcm);
        });
        if (rc) return rc;
        if ((rc = launch(ctx, LWB_KERNEL_SAVE_STATE, k_save_state, g2, b2, 0, dp, (const float *)ctx->x.p))) return rc;
    }
    return LWB_OK;
}

// Any batch: not captured by a prepared batch, which plans it again on every execution.
static int try_generic(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled, lwb_plan *)
{
    *handled = true;
    const BatchExtent &ext = bw.ext;
    if (ext.empty()) return LWB_OK;
    const unsigned C = chains[0].stream->setup->channels;
    std::vector<PlanChain> plan(n_chains);
    for (size_t i = 0; i < n_chains; i++) {
        PlanChain &pc = plan[i];
        pc.c = &chains[i];
        pc.pk.reserve(bw.walks[i].done);
        walk_chain(pc.c, [&](uint32_t, const Geom &g, bool has, uint32_t plen, uint64_t coeff, uint64_t pos) {
            pc.pk.push_back(PlanPacket{g, has ? plen : 0, coeff, pos});
        });
    }
    BatchArenas ar;
    int rc;
    if ((rc = ar.open(ctx, io, ext, C, false)) || (rc = ar.upload(0, ext)) || (rc = run_generic(ctx, plan, io, ar, ext.need_floor0)) ||
        (rc = ar.download(0, bw, 0, n_chains, ext)))
        return rc;
    return ar.finish();
}

