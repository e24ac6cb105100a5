// path_mixed.cuh -- part of the C-ABI translation unit (included by lwb_api.cu, not compiled on its own):
// segmented batches: every chain is cut between the fused long-block kernels, the fused short-block kernels and the
// chain kernel; well-formed 256/2048 chains run in one pass (k_long_s once, then k_short / k_short_g once), the rest
// round by round.
#pragma once

// ---------------------------------------------------------------------------------------------
// Mixed short/long streams (the standard 256/2048 Vorbis shape), and uniform streams of 256-point blocks:
// each chain is cut into segments -- maximal runs of long blocks (n = 2048) go to the fused kernel k_long / k_long_s,
// maximal runs of full-window 256-point blocks to its short-block counterparts k_short / k_short_g, everything else to
// the chain kernel.  Chains that alternate cleanly between long and short segments are executed in ONE PASS (round 0:
// all their long segments, then all their short ones, 128-sample boundary slots in between, see try_mixed); the
// segments of the other chains round by round behind it, handing the overlap state over through the stream's device
// state (PreviousWindowRight) between launches.
// ---------------------------------------------------------------------------------------------
// Static deals (run r -> warp r mod W: k_long_s, k_short) finish with their most loaded warp: order the runs so that
// the W columns carry equal packet counts -- longest first, dealt boustrophedon (row 0 left to right, row 1 right to
// left, ...).  With random run lengths an unordered deal leaves the slowest of 1184 warps a third above the mean.
template <typename Run>
static void balance_static_deal(Run *runs, size_t n, size_t W, std::vector<Run> &tmp)
{
    if (n <= W || W < 2) return;
    uint32_t maxp = 0;
    for (size_t i = 0; i < n; i++) maxp = std::max(maxp, runs[i].n_packets);
    std::vector<size_t> start(maxp + 2, 0);
    for (size_t i = 0; i < n; i++) start[maxp - runs[i].n_packets + 1]++;          // counting sort, descending
    for (size_t k = 1; k < start.size(); k++) start[k] += start[k - 1];
    tmp.resize(n);
    const size_t full_rows = n / W;
    for (size_t i = 0; i < n; i++) {
        const size_t k = start[maxp - runs[i].n_packets]++;
        const size_t row = k / W, col = k % W;
        tmp[(row & 1) && row < full_rows ? row * W + (W - 1 - col) : k] = runs[i];
    }
    std::memcpy(runs, tmp.data(), n * sizeof(Run));
}
// a group of k_short_g: eight runs of one length (the deal above moves it as a unit)
struct ShortGroup { ShortRun r[kShortOct]; uint32_t n_packets; };

static int try_mixed(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled,
                     lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (getenv("LWB_NO_MIXED")) return LWB_OK;
    if (!fused_layout(chains, n_chains, io)) return LWB_OK;
    const bool residue = io->entry != LWB_ENTRY_SPECTRUM;
    const size_t esz = out_format_of(io->out_format).esz;
    unsigned maxc = 1;
    int n1max = 64, n0max = 64, bs0 = -1;
    size_t total_packets = 0, fast_like = 0;
    const float *pack = nullptr, *spack = nullptr, *w_short = nullptr;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_setup *su = c->stream->setup;
        if (su->channels > 8) return LWB_OK;
        // one twiddle pack per launch of each fused kernel (setups with identical tables share theirs, see
        // lwb_setup_create), and one short window for the long kernel's transitional blocks
        const bool long_ok = su->bs1 == kLongBs && su->host.tab[1].pack;
        if (long_ok) {
            if (pack && pack != su->host.tab[1].pack) return LWB_OK;
            pack = su->host.tab[1].pack;
            if (bs0 >= 0 && (bs0 != su->bs0 || w_short != su->host.tab[0].window)) return LWB_OK;
            bs0 = su->bs0;
            w_short = su->host.tab[0].window;
        }
        bool short_ok[2];
        for (int f = 0; f < 2; f++) {
            short_ok[f] = su->host.tab[f].bs == kShortBs && su->host.tab[f].pack && !getenv("LWB_NO_SHORT");
            if (short_ok[f]) {
                if (spack && spack != su->host.tab[f].pack) return LWB_OK;
                spack = su->host.tab[f].pack;
            }
        }
        maxc = std::max<unsigned>(maxc, su->channels);
        n1max = std::max(n1max, 1 << su->bs1);
        n0max = std::max(n0max, 1 << su->bs0);
        total_packets += c->n_packets;
        for (uint32_t k = 0; k < c->n_packets; k++) {
            const uint8_t m = c->mode_numbers[k];
            if (m >= su->n_modes) continue;
            const int f = su->host.mode_blockflag[m];
            if ((f && long_ok) || short_ok[f]) fast_like++;
        }
    }
    // worth it only if the fused kernels get a good share of the packets (every hand-over between the
    // kernels costs a launch): at least half of them
    if (fast_like * 2 < total_packets) return LWB_OK;
    const int bs0e = bs0 >= 0 ? bs0 : kShortBs;
    const int ls_long = (kLongN - (1 << bs0e)) >> 2, pl_short = 1 << (bs0e - 1);
    *handled = true;

    enum { SEG_CHAIN = 0, SEG_LONG = 1, SEG_SHORT = 2 };
    struct Seg { int kind; bool first_short, last_short; uint32_t p0, n; bool has; uint32_t plen; uint64_t coeff, pos; };
    bool chain_sees_long = false;       // the chain kernel's shared memory is sized for what it actually gets
    struct Walk { uint32_t seg0, n_seg; uint32_t boff; size_t slot0; };
    std::vector<Walk> walks(n_chains);
    std::vector<Seg> segs;
    segs.reserve(n_chains * 2);
    struct Pk { bool has; uint32_t plen; uint64_t coeff, pos; };
    std::vector<Pk> pk;
    std::vector<uint8_t> bytes(total_packets * 3 + 16);
    size_t boff = 0, max_rounds = 0;
    const BatchExtent &ext = bw.ext;
    int rc = LWB_OK;
    std::vector<uint8_t> is_l;           // bit0 k_long packet, bit1 follows a short block, bit2 precedes one; bit3 k_short packet
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_setup *su = c->stream->setup;
        Walk &w = walks[i];
        w.boff = (uint32_t)boff;
        // pass 1: geometry + which packets the fused kernel may take (state entering them is empty or 1024)
        if (pk.size() < c->n_packets) { pk.resize(c->n_packets); is_l.resize(c->n_packets); }
        w.seg0 = (uint32_t)segs.size();
        w.n_seg = 0;
        walk_chain(c, [&](uint32_t k, const Geom &g, bool has, uint32_t plen, uint64_t coeff, uint64_t pos) {
            pk[k] = Pk{has, plen, coeff, pos};
            is_l[k] = 0;
            if (g.blockflag && g.n == (uint32_t)kLongN && su->host.tab[1].pack == pack && pack) {
                const bool fs = g.ls != 0, lsf = g.re != g.n;
                if (!has || plen == (fs ? (uint32_t)pl_short : (uint32_t)kLongN2)) is_l[k] = 1 | (fs ? 2 : 0) | (lsf ? 4 : 0);
            } else if (g.n == (uint32_t)kShortN && spack && su->host.tab[g.blockflag].pack == spack && g.ls == 0 &&
                       g.rs == (uint32_t)kShortN2 && g.re == (uint32_t)kShortN && (!has || plen == (uint32_t)kShortN2)) {
                is_l[k] = 8;            // a full-window 256-point block on top of an empty or 128-sample state
            }
            write_mode_bytes(c, k, &bytes[boff + 3 * k]);
        });
        const uint32_t done = bw.walks[i].done;
        boff += (size_t)done * 3;
        if (!done) continue;
        // pass 2: segments.  A fused-kernel run starts at a long block that follows a short one and ends at
        // one that precedes a short one; everything else is handed to the chain kernel.
        uint32_t k = 0;
        while (k < done) {
            uint32_t j = k + 1;
            if (is_l[k] & 1) {
                while (j < done && (is_l[j] & 1) && !(is_l[j - 1] & 4) && !(is_l[j] & 2)) j++;
                segs.push_back(Seg{SEG_LONG, (is_l[k] & 2) != 0, (is_l[j - 1] & 4) != 0, k, j - k, pk[k].has, pk[k].plen, pk[k].coeff,
                                     pk[k].pos});
            } else if (is_l[k] & 8) {
                while (j < done && (is_l[j] & 8)) j++;
                segs.push_back(Seg{SEG_SHORT, false, false, k, j - k, pk[k].has, pk[k].plen, pk[k].coeff, pk[k].pos});
            } else {
                while (j < done && !is_l[j]) j++;
                for (uint32_t q = k; q < j; q++)
                    if (su->host.mode_blockflag[c->mode_numbers[q]]) chain_sees_long = true;
                segs.push_back(Seg{SEG_CHAIN, false, false, k, j - k, pk[k].has, pk[k].plen, pk[k].coeff, pk[k].pos});
            }
            k = j;
        }
        w.n_seg = (uint32_t)segs.size() - w.seg0;
        max_rounds = std::max<size_t>(max_rounds, w.n_seg);
    }
    // One pass instead of rounds: where every chain alternates strictly between long and short segments, the only
    // thing a segment needs from its predecessor is the pl = 128 samples the two blocks overlap in, and the sum
    // x[ls + i] w[i] + prev[i] w[pl-1-i] (audio.rs:1112-1118) does not care which of its two products exists first.
    // So k_long runs ONCE over all long segments -- a run that follows a short block leaves its product in a
    // boundary slot (LongRun::first_short == 2), a run that precedes one leaves its raw right half in another --
    // and k_short then runs ONCE over all short segments, reading the one and completing the other (ShortRun::tail).
    // Per chain: chains that are not such an alternation (a segment for the chain kernel, inconsistent window flags)
    // keep the rounds -- round r + 1 = their segment r -- behind the pass (round 0) of all the others.
    const bool flat_enabled = max_rounds > 1 && !getenv("LWB_MIXED_ROUNDS") && ls_long == kLongLs256;   // (k_long_s exists for blocksize_0 = 256)
    std::vector<uint8_t> chain_flat(n_chains, 0);
    bool flat = false;                                    // some chain takes the pass
    size_t n_slots = 1;                                   // boundary slots of 128 floats: (boundary, channel); slot 0 unused
    size_t rounds_rest = 0;                               // rounds of the chains that do not
    for (size_t i = 0; i < n_chains; i++) {
        const Walk &w = walks[i];
        bool ok = flat_enabled && w.n_seg > 0;
        for (uint32_t q = 0; q < w.n_seg && ok; q++) {
            const Seg &sg = segs[w.seg0 + q];
            if (sg.kind == SEG_CHAIN) ok = false;
            else if (q && sg.kind == segs[w.seg0 + q - 1].kind) ok = false;
            else if (sg.kind == SEG_LONG && ((q && !sg.first_short) || (q + 1 < w.n_seg && !sg.last_short))) ok = false;
        }
        chain_flat[i] = ok;
        if (ok) flat = true;
        else rounds_rest = std::max<size_t>(rounds_rest, w.n_seg);
    }
    // the pass costs three or four launches of its own: not worth it beside the rounds of a batch that is mostly unclean
    {
        size_t pk_flat = 0, pk_all = 0;
        for (size_t i = 0; i < n_chains; i++) {
            pk_all += bw.walks[i].done;
            if (chain_flat[i]) pk_flat += bw.walks[i].done;
        }
        if (!flat_enabled || pk_flat * 2 < pk_all) {
            std::fill(chain_flat.begin(), chain_flat.end(), 0);
            flat = false;
        }
    }
    const size_t round_base = flat ? 1 : 0;               // first round of the chains outside the pass
    // The stream's state row is read by the chain's first segment and written by its last, which now run in no
    // particular order: the old state is moved to slots first (k_row_copy) and the first segment reads those.
    auto needs_precopy = [&](size_t i) { return chain_flat[i] && walks[i].n_seg > 1 && segs[walks[i].seg0].has; };
    auto pre_units = [&](size_t i) {         // slots per channel: a long block on top of a long one overlaps in 1024 samples
        const Seg &sg = segs[walks[i].seg0];
        return (size_t)(sg.kind == SEG_LONG && !sg.first_short ? kLongN2 / kShortN2 : 1);
    };
    size_t n_rc = 0;
    if (flat) {
        for (size_t i = 0; i < n_chains; i++) {
            if (!chain_flat[i]) continue;
            const unsigned C = chains[i].stream->setup->channels;
            walks[i].slot0 = n_slots;
            if (walks[i].n_seg > 1) n_slots += (size_t)(walks[i].n_seg - 1) * C;
            if (needs_precopy(i)) { n_slots += C * pre_units(i); n_rc += C; }       // behind the chain's boundary slots
        }
        max_rounds = round_base + rounds_rest;
    }
    // segments of chain i that round r launches: all of them in round 0 for a chain in the pass, else segment r - round_base
    auto seg_range = [&](size_t i, size_t r, uint32_t *q0, uint32_t *q1) {
        if (chain_flat[i]) { *q0 = 0; *q1 = r == 0 ? walks[i].n_seg : 0; }
        else if (r < round_base) { *q0 = *q1 = 0; }
        else {
            *q0 = (uint32_t)std::min<size_t>(r - round_base, walks[i].n_seg);
            *q1 = (uint32_t)std::min<size_t>(r - round_base + 1, walks[i].n_seg);
        }
    };
    auto round_of = [&](size_t i, uint32_t q) { return chain_flat[i] ? (size_t)0 : round_base + q; };
    const int n1max_all = n1max;         // largest blocksize of the batch (front stages); n1max below sizes the chain kernel
    if (!chain_sees_long) n1max = n0max;
    if (max_rounds) {
        const bool host = io->memory == LWB_MEM_HOST;
        BatchArenas ar;
        if ((rc = ar.open(ctx, io, ext, maxc, true))) return rc;
        char *d_pcm = ar.pcm;
        // host memory: chunks of chains
        const size_t n_chunks = host ? host_chunks((size_t)(ext.c_hi - ext.c_lo) * 4, n_chains) : 1;
        // descriptors of every round: [LongRun...][ChainDesc...][DevPacket (prologue of the long segments)...][mode bytes]
        // A round with few fused-kernel runs leaves most of the SMs x 8 warps idle and lasts as long as its
        // longest run: such rounds cut their runs (each cut costs one extra IMDCT, the primer packet whose
        // right half is all the next piece needs), as the all-long path does.
        const size_t target_runs = (size_t)ctx->sm_count * kLongWarps * 2;
        const size_t target_sruns = (size_t)ctx->sm_count * kShortWarps * 2;
        constexpr uint32_t kMinCutRun = 6, kMinCutShort = 16;       // packets per piece (a cut costs one more transform)
        struct Chunk {
            size_t i0, i1, p0, np_;                      // chains, prologue packets
            BatchExtent ext;
            std::vector<uint32_t> round_cut, round_cut_s;
            std::vector<Step> steps;
        };
        std::vector<Chunk> chunks(n_chunks);
        auto cuts_of = [&](const Chunk &ck, const Seg &sg, size_t r) {
            return sg.kind == SEG_LONG ? std::max<uint32_t>(1, std::min(ck.round_cut[r], sg.n / kMinCutRun))
                                       : std::max<uint32_t>(1, std::min(ck.round_cut_s[r], sg.n / kMinCutShort));
        };
        size_t n_runs = 0, n_sruns = 0, n_cd = 0, n_pro = 0, n_burst = 0;
        // one pass: short segments of fewer than eight packets go to k_short_g, eight of equal length per warp
        const bool bursts = flat && !getenv("LWB_NO_BURSTS");
        for (size_t k = 0; k < n_chunks; k++) {
            Chunk &ck = chunks[k];
            ck.i0 = n_chains * k / n_chunks;
            ck.i1 = n_chains * (k + 1) / n_chunks;
            ck.ext = chunk_extent(io, chains, bw, ck.i0, ck.i1);
            std::vector<size_t> round_long(max_rounds, 0), round_short(max_rounds, 0);
            for (size_t i = ck.i0; i < ck.i1; i++) {
                const unsigned C = chains[i].stream->setup->channels;
                for (uint32_t q = 0; q < walks[i].n_seg; q++) {
                    if (segs[walks[i].seg0 + q].kind == SEG_LONG) round_long[round_of(i, q)] += C;
                    if (segs[walks[i].seg0 + q].kind == SEG_SHORT) round_short[round_of(i, q)] += C;
                }
            }
            ck.round_cut.assign(max_rounds, 1);
            ck.round_cut_s.assign(max_rounds, 1);
            for (size_t r = 0; r < max_rounds; r++) {
                if (round_long[r] && round_long[r] < target_runs)
                    ck.round_cut[r] = (uint32_t)std::min<size_t>(16, (target_runs + round_long[r] - 1) / round_long[r]);
                if (round_short[r] && round_short[r] < target_sruns)
                    ck.round_cut_s[r] = (uint32_t)std::min<size_t>(64, (target_sruns + round_short[r] - 1) / round_short[r]);
            }
            for (size_t i = ck.i0; i < ck.i1; i++)
                for (uint32_t q = 0; q < walks[i].n_seg; q++) {
                    const Seg &sg = segs[walks[i].seg0 + q];
                    if (sg.kind == SEG_LONG) n_runs += (size_t)chains[i].stream->setup->channels * cuts_of(ck, sg, round_of(i, q));
                    else if (sg.kind == SEG_SHORT) {
                        n_sruns += (size_t)chains[i].stream->setup->channels * cuts_of(ck, sg, round_of(i, q));
                        if (bursts && chain_flat[i] && sg.n < (uint32_t)kShortOct) n_burst += chains[i].stream->setup->channels;
                    }
                    else n_cd++;
                    if (residue) n_pro += sg.n;
                }
        }
        // a prepared batch (device memory, spectrum entry) owns its descriptors so that later executions replay them
        const bool cap = plan && !host;
        DevBuf &dbuf = cap ? plan->mix : ctx->cdesc;
        const size_t off_sr = n_runs * sizeof(LongRun), off_cd = off_sr + n_sruns * sizeof(ShortRun), off_pro = off_cd + n_cd * sizeof(ChainDesc);
        const size_t off_rc = off_pro + n_pro * sizeof(DevPacket);
        // burst groups: every length class of every chunk is padded to a multiple of eight runs
        const size_t sg_cap = n_burst ? n_burst + n_chunks * (size_t)(kShortOct * kShortOct) : 0;
        const size_t off_sg = (off_rc + n_rc * sizeof(RowCopy) + 15) & ~(size_t)15;
        const size_t off_by = off_sg + sg_cap * sizeof(ShortRun), total = off_by + boff + 16;
        // boundary slots (device only, not part of the upload); k_long's state copy reads 4 KB wherever it reads
        const size_t off_slots = (total + 511) & ~(size_t)511, slots_bytes = flat ? n_slots * (kShortN2 * 4) + 4096 : 0;
        Staging *st;
        if ((rc = acquire_staging(ctx, total, &st))) return rc;
        if ((rc = ensure(ctx, dbuf, off_slots + slots_bytes))) return rc;
        char *hb = (char *)st->h, *db = (char *)dbuf.p;
        float *d_slots = (float *)(db + off_slots);
        auto slot_of = [&](size_t i, uint32_t boundary, unsigned C, unsigned ch) {      // between segments `boundary` and + 1 of chain i
            return d_slots + (walks[i].slot0 + (size_t)boundary * C + ch) * kShortN2;
        };
        auto pre_slot = [&](size_t i, unsigned C, unsigned ch) {                          // copy of the state the chain starts from
            return d_slots + (walks[i].slot0 + (size_t)(walks[i].n_seg - 1) * C + ch * pre_units(i)) * kShortN2;
        };
        LongRun *h_runs = (LongRun *)hb;
        ShortRun *h_sr = (ShortRun *)(hb + off_sr);
        ChainDesc *h_cd = (ChainDesc *)(hb + off_cd);
        DevPacket *h_pro = (DevPacket *)(hb + off_pro);
        RowCopy *h_rc = (RowCopy *)(hb + off_rc);
        ShortRun *h_sg = (ShortRun *)(hb + off_sg);
        size_t wx = 0, wg = 0;                      // wg: groups written
        std::vector<ShortRun> burst_runs;
        std::vector<ShortGroup> groups, tmp_g;
        std::memcpy(hb + off_by, bytes.data(), boff);
        const float *d_in = ar.coeffs;                           // what the fused kernels and the chain kernel read
        if (residue) {
            if ((rc = ensure(ctx, ctx->spec, (size_t)(ext.c_hi - ext.c_lo) * 4))) return rc;
            d_in = (const float *)ctx->spec.p - ext.c_lo;        // the spectrum: same element offsets as the coefficient arena
        }
        size_t wr = 0, ws = 0, wc = 0, wp = 0;
        std::vector<LongRun> tmp_lr;
        std::vector<ShortRun> tmp_sr;
        // front-stage descriptors of one segment (residue entry)
        auto emit_pro = [&](const lwb_chain *c, const Seg &sg) {
            write_front_packets(c, sg.p0, sg.n, sg.coeff, h_pro + wp);
            wp += sg.n;
        };
        for (Chunk &ck : chunks) {
            ck.p0 = wp;
            for (size_t r = 0; r < max_rounds; r++) {
                const size_t r0 = wr, s0 = ws, c0 = wc, x0 = wx, g0 = wg;
                burst_runs.clear();
                // fused-kernel runs first, longest first (three buckets): the kernel hands runs out in
                // descriptor order, and a 64-packet run started last would be the whole round's tail
                for (int bucket = 0; bucket < 3; bucket++)
                    for (size_t i = ck.i0; i < ck.i1; i++) {
                      uint32_t q0, q1;
                      seg_range(i, r, &q0, &q1);
                      for (uint32_t q = q0; q < q1; q++) {
                        const Seg &sg = segs[walks[i].seg0 + q];
                        if (sg.kind != SEG_LONG) continue;
                        const uint32_t cuts = cuts_of(ck, sg, r), piece = sg.n / cuts;
                        if ((piece >= 32 ? 0 : piece >= 8 ? 1 : 2) != bucket) continue;
                        const lwb_chain *c = &chains[i];
                        const unsigned C = c->stream->setup->channels;
                        // samples packet 0 emits (0 without history; a block after a short one emits 1024 - ls)
                        const size_t first_emit = sg.has ? (sg.first_short ? (size_t)kLongN2 - ls_long : (size_t)kLongN2) : 0;
                        for (unsigned ch = 0; ch < C; ch++) {
                            LongRun *w = h_runs + wr;
                            wr += cuts;
                            channel_run(c, ch, kLongN2, d_in + sg.coeff, d_pcm + sg.pos * esz, esz, sg.n, sg.has, first_emit, cuts, w);
                            LongRun &last = w[cuts - 1], &lr = w[0];         // (one piece: the same run)
                            last.last_short = sg.last_short;
                            if (chain_flat[i] && q + 1 < walks[i].n_seg) last.state_out = slot_of(i, q, C, ch);
                            lr.first_short = sg.first_short;
                            if (chain_flat[i] && q) {   // the short segment in front runs later and completes the overlap
                                lr.first_short = 2;
                                lr.state_out = lr.state_out ? lr.state_out : lr.state;
                                lr.state = slot_of(i, q - 1, C, ch);
                            } else if (needs_precopy(i)) {
                                lr.state_out = lr.state_out ? lr.state_out : lr.state;
                                h_rc[wx++] = RowCopy{lr.state, pre_slot(i, C, ch), (uint32_t)(pre_units(i) * kShortN2 / 4), 0};
                                lr.state = pre_slot(i, C, ch);
                            }
                        }
                        if (residue) emit_pro(c, sg);
                      }
                    }
                // short-block runs: one per channel (and per cut) of every short segment of this round
                for (size_t i = ck.i0; i < ck.i1; i++) {
                  uint32_t q0, q1;
                  seg_range(i, r, &q0, &q1);
                  for (uint32_t q = q0; q < q1; q++) {
                    const Seg &sg = segs[walks[i].seg0 + q];
                    if (sg.kind != SEG_SHORT) continue;
                    const lwb_chain *c = &chains[i];
                    const unsigned C = c->stream->setup->channels;
                    const uint32_t cuts = cuts_of(ck, sg, r);
                    const size_t first_emit = sg.has ? (size_t)kShortN2 : 0;       // samples packet 0 emits
                    const bool burst = bursts && chain_flat[i] && sg.n < (uint32_t)kShortOct;    // (one piece)
                    for (unsigned ch = 0; ch < C; ch++) {
                        ShortRun *w;
                        if (burst) {
                            burst_runs.resize(burst_runs.size() + cuts);
                            w = &burst_runs[burst_runs.size() - cuts];
                        } else {
                            w = h_sr + ws;
                            ws += cuts;
                        }
                        channel_run(c, ch, kShortN2, d_in + sg.coeff, d_pcm + sg.pos * esz, esz, sg.n, sg.has, first_emit, cuts, w);
                        ShortRun &last = w[cuts - 1], &sr = w[0];        // (one piece: the same run)
                        if (chain_flat[i] && q + 1 < walks[i].n_seg) {      // the long block behind has run already
                            last.write_state = 0;
                            last.tail = 1;
                            last.end_ptr = slot_of(i, q, C, ch);
                        }
                        if (chain_flat[i] && q) {       // the long segment in front left its right half in the slot
                            if (!sr.end_ptr) sr.end_ptr = sr.state;
                            sr.state = slot_of(i, q - 1, C, ch);
                        } else if (needs_precopy(i)) {
                            if (!sr.end_ptr) sr.end_ptr = sr.state;
                            h_rc[wx++] = RowCopy{sr.state, pre_slot(i, C, ch), (uint32_t)(kShortN2 / 4), 0};
                            sr.state = pre_slot(i, C, ch);
                        }
                    }
                    if (residue) emit_pro(c, sg);
                  }
                }
                for (size_t i = ck.i0; i < ck.i1; i++) {
                    uint32_t q0, q1;
                    seg_range(i, r, &q0, &q1);
                    if (q0 >= q1) continue;
                    const Seg &sg = segs[walks[i].seg0 + q0];
                    if (sg.kind != SEG_CHAIN) continue;
                    const lwb_chain *c = &chains[i];
                    if (residue) emit_pro(c, sg);
                    chain_desc(c, sg.p0, sg.n, sg.has, sg.plen, sg.coeff, sg.pos, walks[i].boff + 3 * sg.p0, &h_cd[wc++]);
                }
                if (!burst_runs.empty()) {
                    // length classes, longest first, each padded with dummies (in == nullptr) to whole groups
                    groups.clear();
                    for (uint32_t len = kShortOct; len-- > 1;) {
                        size_t in_class = 0;
                        for (const ShortRun &br : burst_runs) {
                            if (br.n_packets != len) continue;
                            if (in_class % kShortOct == 0) {
                                groups.emplace_back();
                                std::memset(&groups.back(), 0, sizeof(ShortGroup));
                                groups.back().n_packets = len;
                                for (int k = 0; k < kShortOct; k++) groups.back().r[k].n_packets = len;
                            }
                            groups.back().r[in_class++ % kShortOct] = br;
                        }
                    }
                    const size_t Wg = (size_t)static_deal_grid(groups.size(), kShortWarps, ctx->sm_count) * kShortWarps;
                    if (!getenv("LWB_NO_BALANCE")) balance_static_deal(groups.data(), groups.size(), Wg, tmp_g);
                    if ((wg + groups.size()) * kShortOct > sg_cap) return fail(ctx, LWB_ERR_INVALID, "burst group area too small");
                    for (const ShortGroup &gr : groups) std::memcpy(h_sg + (wg++) * kShortOct, gr.r, sizeof(gr.r));
                }
                const size_t nr = wr - r0, ns = ws - s0;
                if (flat && r == 0 && !getenv("LWB_NO_BALANCE")) {
                    balance_static_deal(h_runs + r0, nr, (size_t)static_deal_grid(nr, kLongWarps, ctx->sm_count) * kLongWarps, tmp_lr);
                    balance_static_deal(h_sr + s0, ns, (size_t)static_deal_grid(ns, kShortWarps, ctx->sm_count) * kShortWarps, tmp_sr);
                }
                // the round's launches: the row copies go before k_long_s, and the short kernels complete the boundary
                // slots k_long_s left
                if (nr && kLongNB != 1) return fail(ctx, LWB_ERR_INVALID, "mixed path needs one run per warp");
                auto step = [&](int kernel, size_t off, size_t n, const float *pk) {
                    if (n) ck.steps.push_back(Step{kernel, db + off, n, pk});
                };
                step(LWB_KERNEL_ROW_COPY, off_rc + x0 * sizeof(RowCopy), wx - x0, nullptr);
                step(flat && r == 0 ? LWB_KERNEL_LONG_S : LWB_KERNEL_LONG, r0 * sizeof(LongRun), nr, pack);
                step(LWB_KERNEL_SHORT, off_sr + s0 * sizeof(ShortRun), ns, spack);
                step(LWB_KERNEL_SHORT_G, off_sg + g0 * kShortOct * sizeof(ShortRun), wg - g0, spack);
                step(LWB_KERNEL_CHAIN, off_cd + c0 * sizeof(ChainDesc), wc - c0, nullptr);
            }
            ck.np_ = wp - ck.p0;
        }
        if ((rc = upload_staging(ctx, st, hb, db, total, ctx->stream))) return rc;
        StepArgs args;
        args.pcm = d_pcm;
        args.out_format = io->out_format;
        args.w_short = w_short;
        args.ls = ls_long;
        args.chain = chain_shape(maxc, n1max, false);
        args.bytes = (const uint8_t *)db + off_by;
        args.coeffs = d_in;                     // (residue entry: the front stages run first, the chain kernel sees a spectrum)
        FrontStages fs = front_stages_of(ext, maxc, n1max_all, n_pro);         // (residue entry: every packet of the batch, chunk by chunk)
        fs.pk = (const DevPacket *)(db + off_pro);
        if (fs.n) fs.fast = front_stages_fast(ctx, ar, fs, h_pro);
        for (size_t k = 0; k < n_chunks; k++) {
            Chunk &ck = chunks[k];
            if (ck.ext.empty()) continue;
            if ((rc = ar.upload(k, ck.ext)) || (ck.np_ && (rc = front_stages_launch(ctx, ar, fs, ck.p0, ck.np_))) ||
                (rc = run_steps(ctx, args, ck.steps)) || (rc = ar.download(k, chains, bw, ck.i0, ck.i1, ck.ext)))
                return rc;
        }
        if (cap) capture(plan, gen_at_entry, fs, args, std::move(chunks[0].steps));
        if ((rc = ar.finish())) return rc;
    }
    return LWB_OK;
}

