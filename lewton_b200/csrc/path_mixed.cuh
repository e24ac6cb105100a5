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
// all their long segments, then all their short ones, 128-sample boundary slots in between, see MixedSchedule); the
// segments of the other chains round by round behind it, handing the overlap state over through the stream's device
// state (PreviousWindowRight) between launches.  Stages: mixed_shape, segment_chain, MixedSchedule, mixed_layout, MixedWriter.
// ---------------------------------------------------------------------------------------------

// What the launches of a segmented batch share: one twiddle pack per fused kernel (setups with identical tables share
// theirs, see lwb_setup_create) and one short window for k_long's transitional blocks.
struct MixedShape {
    const float *pack = nullptr, *spack = nullptr, *w_short = nullptr;
    int bs0 = -1, n1max = 64, n0max = 64, ls_long = 0, pl_short = 0;
    unsigned maxc = 1;
    size_t total_packets = 0;
};

// The shape of a batch, or false if the segmented path does not take it: more than 8 channels, two packs for one fused
// kernel, or fewer than half the packets for the fused kernels (every hand-over between the kernels costs a launch).
static bool mixed_shape(const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, bool no_short, MixedShape *sh)
{
    if (!fused_layout(chains, n_chains, io)) return false;
    size_t fast_like = 0;
    for (size_t i = 0; i < n_chains; i++) {
        const lwb_chain *c = &chains[i];
        const lwb_setup *su = c->stream->setup;
        if (su->channels > 8) return false;
        const bool long_ok = su->bs1 == kLongBs && su->host.tab[1].pack;
        if (long_ok) {
            if (sh->pack && sh->pack != su->host.tab[1].pack) return false;
            sh->pack = su->host.tab[1].pack;
            if (sh->bs0 >= 0 && (sh->bs0 != su->bs0 || sh->w_short != su->host.tab[0].window)) return false;
            sh->bs0 = su->bs0;
            sh->w_short = su->host.tab[0].window;
        }
        bool short_ok[2];
        for (int f = 0; f < 2; f++) {
            short_ok[f] = su->host.tab[f].bs == kShortBs && su->host.tab[f].pack && !no_short;
            if (short_ok[f]) {
                if (sh->spack && sh->spack != su->host.tab[f].pack) return false;
                sh->spack = su->host.tab[f].pack;
            }
        }
        sh->maxc = std::max<unsigned>(sh->maxc, su->channels);
        sh->n1max = std::max(sh->n1max, 1 << su->bs1);
        sh->n0max = std::max(sh->n0max, 1 << su->bs0);
        sh->total_packets += c->n_packets;
        for (uint32_t k = 0; k < c->n_packets; k++) {
            const uint8_t m = c->mode_numbers[k];
            if (m >= su->n_modes) continue;
            const int f = su->host.mode_blockflag[m];
            if ((f && long_ok) || short_ok[f]) fast_like++;
        }
    }
    if (fast_like * 2 < sh->total_packets) return false;
    const int bs0e = sh->bs0 >= 0 ? sh->bs0 : kShortBs;
    sh->ls_long = (kLongN - (1 << bs0e)) >> 2;
    sh->pl_short = 1 << (bs0e - 1);
    return true;
}

enum SegKind : uint8_t { SEG_CHAIN, SEG_LONG, SEG_SHORT };
// Packets [p0, p0 + n) of a chain for one kernel, with the state entering them, their coefficient offset and the samples
// before them; k_long: the first follows a short block (first_short), the last precedes one (last_short).
struct MixedSeg { SegKind kind; bool first_short, last_short; uint32_t p0, n; bool has; uint32_t plen; uint64_t coeff, pos; };

// One pass instead of rounds: where every chain alternates strictly between long and short segments, the only thing a
// segment needs from its predecessor is the pl = 128 samples the two blocks overlap in, and the sum
// x[ls + i] w[i] + prev[i] w[pl-1-i] (audio.rs:1112-1118) does not care which of its two products exists first.  So
// k_long runs ONCE over all long segments -- a run that follows a short block leaves its product in a boundary slot
// (LongRun::first_short == 2), a run that precedes one leaves its raw right half in another -- and k_short then runs
// ONCE over all short segments, reading the one and completing the other (ShortRun::tail).  Per chain: chains that are
// not such an alternation (a segment for the chain kernel, inconsistent window flags) keep the rounds -- round r + 1 =
// their segment r -- behind the pass (round 0) of all the others.
struct MixedSchedule {
    struct Chain {
        uint32_t seg0 = 0, n_seg = 0, boff = 0;   // segments segs[seg0, seg0 + n_seg), mode bytes at boff
        size_t slot0 = 0;                         // first boundary slot
        bool pass = false;                        // the chain takes the pass
    };
    std::vector<Chain> chain;
    std::vector<MixedSeg> segs;
    size_t round_base = 0, max_rounds = 0;        // round_base: first round of the chains outside the pass
    size_t n_slots = 1;                           // boundary slots of 128 floats: (boundary, channel); slot 0 unused
    size_t n_rc = 0;                              // state-row copies in front of the pass
    bool bursts = false;                          // short segments of fewer than eight packets in the pass go to k_short_g
    bool pass() const { return round_base != 0; }
    const MixedSeg &seg(size_t i, uint32_t q) const { return segs[chain[i].seg0 + q]; }
    bool burst(size_t i, const MixedSeg &sg) const { return bursts && chain[i].pass && sg.n < (uint32_t)kShortOct; }
    // segments [q0, q1) of chain i in round r: all of them in round 0 for a chain in the pass, else segment r - round_base
    std::pair<uint32_t, uint32_t> round_segs(size_t i, size_t r) const
    {
        const Chain &w = chain[i];
        if (w.pass) return {0, r == 0 ? w.n_seg : 0};
        const uint32_t q = r < round_base ? w.n_seg : (uint32_t)std::min<size_t>(r - round_base, w.n_seg);
        return {q, std::min(q + 1, w.n_seg)};
    }
    size_t round_of(size_t i, uint32_t q) const { return chain[i].pass ? 0 : round_base + q; }
    // The stream's state row is read by the chain's first segment and written by its last, which now run in no
    // particular order: the old state is moved to slots first (k_row_copy) and the first segment reads those.
    bool needs_precopy(size_t i) const { return chain[i].pass && chain[i].n_seg > 1 && seg(i, 0).has; }
    // slots per channel of the copy: a long block on top of a long one overlaps in 1024 samples
    size_t pre_units(size_t i) const { return seg(i, 0).kind == SEG_LONG && !seg(i, 0).first_short ? kLongN2 / kShortN2 : 1; }
    // the slot between segments `boundary` and + 1 of chain i (C channels) for channel ch, and that of its state copy
    size_t slot_of(size_t i, uint32_t boundary, unsigned C, unsigned ch) const { return chain[i].slot0 + (size_t)boundary * C + ch; }
    size_t pre_slot(size_t i, unsigned C, unsigned ch) const { return slot_of(i, chain[i].n_seg - 1, C, 0) + ch * pre_units(i); }
    // Chooses the chains that take the pass (none unless `enabled`) and sizes the rounds and slots.  The pass costs three
    // or four launches of its own: beside the rounds of a mostly unclean batch it is not worth it.
    void plan(const lwb_chain *chains, const BatchWalk &bw, bool enabled, bool with_bursts)
    {
        for (const Chain &w : chain) max_rounds = std::max<size_t>(max_rounds, w.n_seg);
        size_t rounds_rest = 0, pk_pass = 0, pk_all = 0;
        for (size_t i = 0; i < chain.size(); i++) {
            Chain &w = chain[i];
            bool ok = enabled && max_rounds > 1 && w.n_seg > 0;
            for (uint32_t q = 0; q < w.n_seg && ok; q++) {
                const MixedSeg &sg = seg(i, q);
                if (sg.kind == SEG_CHAIN) ok = false;
                else if (q && sg.kind == seg(i, q - 1).kind) ok = false;
                else if (sg.kind == SEG_LONG && ((q && !sg.first_short) || (q + 1 < w.n_seg && !sg.last_short))) ok = false;
            }
            w.pass = ok;
            if (ok) pk_pass += bw.walks[i].done;
            else rounds_rest = std::max<size_t>(rounds_rest, w.n_seg);
            pk_all += bw.walks[i].done;
        }
        if (!pk_pass || pk_pass * 2 < pk_all) {
            for (Chain &w : chain) w.pass = false;
            return;
        }
        round_base = 1;
        max_rounds = round_base + rounds_rest;
        bursts = with_bursts;
        for (size_t i = 0; i < chain.size(); i++) {
            if (!chain[i].pass) continue;
            const unsigned C = chains[i].stream->setup->channels;
            chain[i].slot0 = n_slots;
            n_slots += (size_t)(chain[i].n_seg - 1) * C;
            if (needs_precopy(i)) {                 // behind the chain's boundary slots
                n_slots += C * pre_units(i);
                n_rc += C;
            }
        }
    }
};

// Cuts the packets chain c decodes (returned) into segments: the next chain of sc, its mode bytes at bytes + boff.  A
// k_long run starts at a long block that follows a short one and ends at one that precedes a short one; the chain
// kernel takes what neither fused kernel takes (*chain_sees_long: a long block among it).  pk: scratch.
static uint32_t segment_chain(const lwb_chain *c, const MixedShape &sh, size_t boff, uint8_t *bytes, std::vector<MixedSeg> &pk, MixedSchedule &sc,
                              bool *chain_sees_long)
{
    const lwb_setup *su = c->stream->setup;
    if (pk.size() < c->n_packets) pk.resize(c->n_packets);
    sc.chain.push_back(MixedSchedule::Chain{(uint32_t)sc.segs.size(), 0, (uint32_t)boff});
    const uint32_t done = walk_chain(c, [&](uint32_t k, const Geom &g, bool has, uint32_t plen, uint64_t coeff, uint64_t pos) {
        MixedSeg &p = pk[k] = MixedSeg{SEG_CHAIN, false, false, k, 1, has, plen, coeff, pos};
        // A long block after a short one of the same size (blocksize_0 == blocksize_1: ls == 0, slope_sel == 0) slopes its
        // whole left half with tab[0]'s window (audio.rs:1059-1088), which k_long's pack holds only when both tables are
        // the same (the context shares equal tables).
        const bool left_ok = g.ls != 0 || g.slope_sel || su->host.tab[0].pack == su->host.tab[1].pack;
        if (g.blockflag && g.n == (uint32_t)kLongN && su->host.tab[1].pack == sh.pack && sh.pack && left_ok) {
            const bool fs = g.ls != 0;
            if (!has || plen == (fs ? (uint32_t)sh.pl_short : (uint32_t)kLongN2)) {     // on the state the block before leaves
                p.kind = SEG_LONG;
                p.first_short = fs;
                p.last_short = g.re != g.n;
            }
        } else if (g.n == (uint32_t)kShortN && sh.spack && su->host.tab[g.blockflag].pack == sh.spack && g.ls == 0 &&
                   g.rs == (uint32_t)kShortN2 && g.re == (uint32_t)kShortN && (!has || plen == (uint32_t)kShortN2)) {
            p.kind = SEG_SHORT;         // a full-window 256-point block on top of an empty or 128-sample state
        }
        write_mode_bytes(c, k, bytes + boff + 3 * k);
    }).done;
    for (uint32_t k = 0, j; k < done; k = j) {
        const SegKind kind = pk[k].kind;
        for (j = k + 1; j < done && pk[j].kind == kind; j++)
            if (kind == SEG_LONG && (pk[j - 1].last_short || pk[j].first_short)) break;
        if (kind == SEG_CHAIN)
            for (uint32_t q = k; q < j; q++)
                if (su->host.mode_blockflag[c->mode_numbers[q]]) *chain_sees_long = true;
        MixedSeg &sg = sc.segs.emplace_back(pk[k]);
        sg.n = j - k;
        sg.last_short = pk[j - 1].last_short;
        sc.chain.back().n_seg++;
    }
    return done;
}

// Chains [i0, i1), one chunk of a host-memory batch.  A round with few fused-kernel runs leaves most of the SMs x 8 warps
// idle and lasts as long as its longest run: such rounds cut their runs (each cut costs one extra IMDCT, the primer
// packet whose right half is all the next piece needs), as the all-long path does.
struct MixedChunk {
    size_t i0, i1, p0, np_;                      // chains, prologue packets
    BatchExtent ext;
    std::vector<uint32_t> round_cut, round_cut_s;      // at most this many pieces per long / short segment of round r
    std::vector<Step> steps;
    uint32_t cuts(const MixedSeg &sg, size_t r) const
    {
        constexpr uint32_t kMinCutRun = 6, kMinCutShort = 16;       // packets per piece (a cut costs one more transform)
        return sg.kind == SEG_LONG ? std::max<uint32_t>(1, std::min(round_cut[r], sg.n / kMinCutRun))
                                   : std::max<uint32_t>(1, std::min(round_cut_s[r], sg.n / kMinCutShort));
    }
};

// The descriptor buffer, uploaded as one: [LongRun][ShortRun][ChainDesc][DevPacket (front stages)][RowCopy][burst groups]
// [mode bytes], then the boundary slots (device only).  sg_cap: the burst runs the group area holds.
struct MixedLayout { size_t off_sr, off_cd, off_pro, off_rc, off_sg, off_by, total, sg_cap, off_slots, slots_bytes; };

// The chunks of chains, each round's cuts and the layout of the descriptor buffer, with n_bytes of mode bytes.
static MixedLayout mixed_layout(const lwb_ctx *ctx, const lwb_chain *chains, const lwb_batch_io *io, const BatchWalk &bw,
                                const MixedSchedule &sc, size_t n_bytes, std::vector<MixedChunk> &chunks)
{
    const size_t target_runs = (size_t)ctx->sm_count * kLongWarps * 2, target_sruns = (size_t)ctx->sm_count * kShortWarps * 2;
    const size_t n_chains = sc.chain.size(), n_chunks = chunks.size(), R = sc.max_rounds;
    size_t n_runs = 0, n_sruns = 0, n_cd = 0, n_pro = 0, n_burst = 0;
    for (size_t k = 0; k < n_chunks; k++) {
        MixedChunk &ck = chunks[k];
        ck.i0 = n_chains * k / n_chunks;
        ck.i1 = n_chains * (k + 1) / n_chunks;
        ck.ext = chunk_extent(io, chains, bw, ck.i0, ck.i1);
        std::vector<size_t> round_long(R, 0), round_short(R, 0);
        for (size_t i = ck.i0; i < ck.i1; i++)
            for (uint32_t q = 0; q < sc.chain[i].n_seg; q++)
                if (sc.seg(i, q).kind != SEG_CHAIN)
                    (sc.seg(i, q).kind == SEG_LONG ? round_long : round_short)[sc.round_of(i, q)] += chains[i].stream->setup->channels;
        ck.round_cut.assign(R, 1);
        ck.round_cut_s.assign(R, 1);
        for (size_t r = 0; r < R; r++) {
            if (round_long[r] && round_long[r] < target_runs)
                ck.round_cut[r] = (uint32_t)std::min<size_t>(16, (target_runs + round_long[r] - 1) / round_long[r]);
            if (round_short[r] && round_short[r] < target_sruns)
                ck.round_cut_s[r] = (uint32_t)std::min<size_t>(64, (target_sruns + round_short[r] - 1) / round_short[r]);
        }
        for (size_t i = ck.i0; i < ck.i1; i++)
            for (uint32_t q = 0; q < sc.chain[i].n_seg; q++) {
                const MixedSeg &sg = sc.seg(i, q);
                const unsigned C = chains[i].stream->setup->channels;
                if (sg.kind == SEG_LONG) n_runs += (size_t)C * ck.cuts(sg, sc.round_of(i, q));
                else if (sg.kind == SEG_SHORT) n_sruns += (size_t)C * ck.cuts(sg, sc.round_of(i, q));
                else n_cd++;
                if (sg.kind == SEG_SHORT && sc.burst(i, sg)) n_burst += C;
                if (io->entry != LWB_ENTRY_SPECTRUM) n_pro += sg.n;
            }
    }
    MixedLayout ly;
    ly.off_sr = n_runs * sizeof(LongRun);
    ly.off_cd = ly.off_sr + n_sruns * sizeof(ShortRun);
    ly.off_pro = ly.off_cd + n_cd * sizeof(ChainDesc);
    ly.off_rc = ly.off_pro + n_pro * sizeof(DevPacket);
    // burst groups: every length class of every chunk is padded to a multiple of eight runs
    ly.sg_cap = n_burst ? n_burst + n_chunks * (size_t)(kShortOct * kShortOct) : 0;
    ly.off_sg = (ly.off_rc + sc.n_rc * sizeof(RowCopy) + 15) & ~(size_t)15;
    ly.off_by = ly.off_sg + ly.sg_cap * sizeof(ShortRun);
    ly.total = ly.off_by + n_bytes + 16;
    // k_long's state copy reads 4 KB wherever it reads
    ly.off_slots = (ly.total + 511) & ~(size_t)511;
    ly.slots_bytes = sc.pass() ? sc.n_slots * (kShortN2 * 4) + 4096 : 0;
    return ly;
}

// Writes the descriptors of every round into the staged buffer hb (laid out by ly) and records each round's steps.
// wr, ws, wc, wp, wx, wg: the LongRuns, ShortRuns, ChainDescs, DevPackets, RowCopys and burst groups written so far.
struct MixedWriter {
    const lwb_chain *chains;
    const MixedSchedule &sc;
    const MixedShape &sh;
    const MixedLayout &ly;
    char *hb, *db, *pcm;              // the staged descriptor buffer, its device copy and the PCM arena
    const float *in;                  // what the fused kernels and the chain kernel read
    size_t esz;
    bool residue, balance;
    size_t wr = 0, ws = 0, wc = 0, wp = 0, wx = 0, wg = 0;
    std::vector<ShortRun> burst_runs;
    float *slot(size_t idx) const { return (float *)(db + ly.off_slots) + idx * kShortN2; }
    void front(const lwb_chain *c, const MixedSeg &sg)          // front-stage descriptors of one segment (residue entry)
    {
        if (!residue) return;
        write_front_packets(c, sg.p0, sg.n, sg.coeff, (DevPacket *)(hb + ly.off_pro) + wp);
        wp += sg.n;
    }
    // In the pass, the first piece of a run of segment q reads the boundary slot in front or, for the chain's first
    // segment, a copy of the state row, which the run still stores to (`end`, unless already set).
    template <typename Run>
    void read_slot(Run &first, float *&end, size_t i, uint32_t q, unsigned C, unsigned ch)
    {
        if (!(sc.chain[i].pass && q) && !sc.needs_precopy(i)) return;
        if (!end) end = first.state;
        float *from = slot(q ? sc.slot_of(i, q - 1, C, ch) : sc.pre_slot(i, C, ch));
        if (!q) ((RowCopy *)(hb + ly.off_rc))[wx++] = RowCopy{first.state, from, sc.pre_units(i) * kShortN2 * sizeof(float)};
        first.state = from;
    }
    // k_long's runs of long segment q of chain i.  In the pass, a run after a short segment leaves its left slope in the
    // slot in front (first_short == 2) for that segment to complete, a run before one its right half in the slot behind.
    void long_seg(size_t i, uint32_t q, uint32_t cuts)
    {
        const lwb_chain *c = &chains[i];
        const MixedSeg &sg = sc.seg(i, q);
        const unsigned C = c->stream->setup->channels;
        const bool pass = sc.chain[i].pass;
        // samples packet 0 emits (0 without history; a block after a short one emits 1024 - ls)
        const size_t first_emit = sg.has ? (sg.first_short ? (size_t)kLongN2 - sh.ls_long : (size_t)kLongN2) : 0;
        for (unsigned ch = 0; ch < C; ch++) {
            LongRun *w = (LongRun *)hb + wr;
            wr += cuts;
            channel_run(c, ch, kLongN2, in + sg.coeff, pcm + sg.pos * esz, esz, sg.n, sg.has, first_emit, cuts, w);
            LongRun &last = w[cuts - 1], &lr = w[0];         // (one piece: the same run)
            last.last_short = sg.last_short;
            if (pass && q + 1 < sc.chain[i].n_seg) last.state_out = slot(sc.slot_of(i, q, C, ch));
            lr.first_short = pass && q ? 2 : sg.first_short;
            read_slot(lr, lr.state_out, i, q, C, ch);
        }
        front(c, sg);
    }
    // k_short's runs of short segment q of chain i, or a burst's for k_short_g (grouped by the round).  In the pass, a run
    // before a long segment completes the overlap it left in the slot behind (tail); after one, it reads the slot in front.
    void short_seg(size_t i, uint32_t q, uint32_t cuts)
    {
        const lwb_chain *c = &chains[i];
        const MixedSeg &sg = sc.seg(i, q);
        const unsigned C = c->stream->setup->channels;
        const bool pass = sc.chain[i].pass, burst = sc.burst(i, sg);      // (a burst is one piece)
        const size_t first_emit = sg.has ? (size_t)kShortN2 : 0;         // samples packet 0 emits
        for (unsigned ch = 0; ch < C; ch++) {
            ShortRun *w = (ShortRun *)(hb + ly.off_sr) + ws;
            if (burst) w = &burst_runs.emplace_back();
            else ws += cuts;
            channel_run(c, ch, kShortN2, in + sg.coeff, pcm + sg.pos * esz, esz, sg.n, sg.has, first_emit, cuts, w);
            ShortRun &last = w[cuts - 1];                    // (one piece: the same run as w[0])
            if (pass && q + 1 < sc.chain[i].n_seg) {         // the long block behind has run already
                last.write_state = 0;
                last.tail = 1;
                last.end_ptr = slot(sc.slot_of(i, q, C, ch));
            }
            read_slot(w[0], w[0].end_ptr, i, q, C, ch);
        }
        front(c, sg);
    }
    // The descriptors of round r of chunk ck, and its launches: the row copies go before k_long_s, and the short kernels
    // complete the boundary slots k_long_s left.
    int round(lwb_ctx *ctx, MixedChunk &ck, size_t r)
    {
        const size_t r0 = wr, s0 = ws, c0 = wc, x0 = wx, g0 = wg;
        burst_runs.clear();
        // fused-kernel runs first, longest first (three buckets): the kernel hands runs out in descriptor order, and a
        // 64-packet run started last would be the whole round's tail
        for (int bucket = 0; bucket < 3; bucket++)
            for (size_t i = ck.i0; i < ck.i1; i++)
                for (auto [q, q1] = sc.round_segs(i, r); q < q1; q++) {
                    const MixedSeg &sg = sc.seg(i, q);
                    const uint32_t cuts = ck.cuts(sg, r), piece = sg.n / cuts;
                    if (sg.kind == SEG_LONG && (piece >= 32 ? 0 : piece >= 8 ? 1 : 2) == bucket) long_seg(i, q, cuts);
                }
        // short-block runs: one per channel (and per cut) of every short segment of this round
        for (size_t i = ck.i0; i < ck.i1; i++)
            for (auto [q, q1] = sc.round_segs(i, r); q < q1; q++)
                if (sc.seg(i, q).kind == SEG_SHORT) short_seg(i, q, ck.cuts(sc.seg(i, q), r));
        for (size_t i = ck.i0; i < ck.i1; i++)
            for (auto [q, q1] = sc.round_segs(i, r); q < q1; q++)
                if (const MixedSeg &sg = sc.seg(i, q); sg.kind == SEG_CHAIN) {
                    front(&chains[i], sg);
                    chain_desc(&chains[i], sg.p0, sg.n, sg.has, sg.plen, sg.coeff, sg.pos, sc.chain[i].boff + 3 * sg.p0, (ChainDesc *)(hb + ly.off_cd) + wc++);
                }
        if (!burst_runs.empty()) {
            // dummies: in == nullptr
            auto groups = group_runs<kShortOct>(burst_runs, kShortOct, [](const ShortRun &first) { ShortRun d{}; d.n_packets = first.n_packets; return d; });
            if (balance) balance_static_deal(groups.data(), groups.size(), kShortWarps, ctx->sm_count);
            if ((wg + groups.size()) * kShortOct > ly.sg_cap) return fail(ctx, LWB_ERR_INVALID, "burst group area too small");
            for (const auto &gr : groups) std::memcpy((ShortRun *)(hb + ly.off_sg) + (wg++) * kShortOct, gr.r, sizeof(gr.r));
        }
        const size_t nr = wr - r0, ns = ws - s0;
        if (sc.pass() && r == 0 && balance) {
            balance_static_deal((LongRun *)hb + r0, nr, kLongWarps, ctx->sm_count);
            balance_static_deal((ShortRun *)(hb + ly.off_sr) + s0, ns, kShortWarps, ctx->sm_count);
        }
        if (nr && kLongNB != 1) return fail(ctx, LWB_ERR_INVALID, "mixed path needs one run per warp");
        for (const Step &s : {Step{LWB_KERNEL_ROW_COPY, db + ly.off_rc + x0 * sizeof(RowCopy), wx - x0, nullptr},
                              Step{sc.pass() && r == 0 ? LWB_KERNEL_LONG_S : LWB_KERNEL_LONG, db + r0 * sizeof(LongRun), nr, sh.pack},
                              Step{LWB_KERNEL_SHORT, db + ly.off_sr + s0 * sizeof(ShortRun), ns, sh.spack},
                              Step{LWB_KERNEL_SHORT_G, db + ly.off_sg + g0 * kShortOct * sizeof(ShortRun), wg - g0, sh.spack},
                              Step{LWB_KERNEL_CHAIN, db + ly.off_cd + c0 * sizeof(ChainDesc), wc - c0, nullptr}})
            if (s.n) ck.steps.push_back(s);
        return LWB_OK;
    }
};

static int try_mixed(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, const BatchWalk &bw, bool *handled,
                     lwb_plan *plan)
{
    *handled = false;
    const uint64_t gen_at_entry = ctx->state_gen;
    if (getenv("LWB_NO_MIXED")) return LWB_OK;
    // test switches: no k_short, rounds instead of the pass, bursts on k_short, runs dealt in descriptor order
    const bool no_short = getenv("LWB_NO_SHORT"), rounds = getenv("LWB_MIXED_ROUNDS"), no_bursts = getenv("LWB_NO_BURSTS"), no_balance = getenv("LWB_NO_BALANCE");
    MixedShape sh;
    if (!mixed_shape(chains, n_chains, io, no_short, &sh)) return LWB_OK;
    *handled = true;
    MixedSchedule sc;
    sc.chain.reserve(n_chains);
    sc.segs.reserve(n_chains * 2);
    std::vector<MixedSeg> pk;
    std::vector<uint8_t> bytes(sh.total_packets * 3 + 16);
    size_t boff = 0;
    bool chain_sees_long = false;       // the chain kernel's shared memory is sized for what it actually gets
    for (size_t i = 0; i < n_chains; i++) boff += 3 * (size_t)segment_chain(&chains[i], sh, boff, bytes.data(), pk, sc, &chain_sees_long);
    sc.plan(chains, bw, !rounds && sh.ls_long == kLongLs256, !no_bursts);       // (k_long_s exists for blocksize_0 = 256)
    if (!sc.max_rounds) return LWB_OK;
    const bool host = io->memory == LWB_MEM_HOST, residue = io->entry != LWB_ENTRY_SPECTRUM;
    const BatchExtent &ext = bw.ext;
    int rc;
    BatchArenas ar;
    if ((rc = ar.open(ctx, io, ext, sh.maxc, true))) return rc;
    std::vector<MixedChunk> chunks(host ? host_chunks((size_t)(ext.c_hi - ext.c_lo) * 4, n_chains) : 1);
    const MixedLayout ly = mixed_layout(ctx, chains, io, bw, sc, boff, chunks);
    // a prepared batch (device memory) owns its descriptors so that later executions replay them
    const bool cap = plan && !host;
    DevBuf &dbuf = cap ? plan->desc : ctx->cdesc;
    Staging *st;
    if ((rc = acquire_staging(ctx, ly.total, &st)) || (rc = ensure(ctx, dbuf, ly.off_slots + ly.slots_bytes))) return rc;
    char *hb = (char *)st->h, *db = (char *)dbuf.p;
    std::memcpy(hb + ly.off_by, bytes.data(), boff);
    const float *d_in = ar.coeffs;
    if (residue) {
        if ((rc = ensure(ctx, ctx->spec, (size_t)(ext.c_hi - ext.c_lo) * 4))) return rc;
        d_in = (const float *)ctx->spec.p - ext.c_lo;        // the spectrum: same element offsets as the coefficient arena
    }
    MixedWriter wt{chains, sc, sh, ly, hb, db, ar.pcm, d_in, out_format_of(io->out_format).esz, residue, !no_balance};
    for (MixedChunk &ck : chunks) {
        ck.p0 = wt.wp;
        for (size_t r = 0; r < sc.max_rounds; r++)
            if ((rc = wt.round(ctx, ck, r))) return rc;
        ck.np_ = wt.wp - ck.p0;
    }
    if ((rc = upload_staging(ctx, st, hb, db, ly.total, ctx->stream))) return rc;
    StepArgs args;
    args.pcm = ar.pcm;
    args.out_format = io->out_format;
    args.w_short = sh.w_short;
    args.ls = sh.ls_long;
    args.chain = chain_shape(sh.maxc, chain_sees_long ? sh.n1max : sh.n0max, false);
    args.bytes = (const uint8_t *)db + ly.off_by;
    args.coeffs = d_in;                     // (residue entry: the front stages run first, the chain kernel sees a spectrum)
    FrontStages fs = front_stages_of(ext, sh.maxc, sh.n1max, wt.wp);        // (residue entry: every packet of the batch, chunk by chunk)
    fs.pk = (const DevPacket *)(db + ly.off_pro);
    if (fs.n) fs.fast = front_stages_fast(ctx, ar, fs, (const DevPacket *)(hb + ly.off_pro));
    for (size_t k = 0; k < chunks.size(); k++) {
        MixedChunk &ck = chunks[k];
        if (ck.ext.empty()) continue;
        if ((rc = ar.upload(k, ck.ext)) || (ck.np_ && (rc = front_stages_launch(ctx, ar, fs, ck.p0, ck.np_))) ||
            (rc = run_steps(ctx, args, ck.steps)) || (rc = ar.download(k, bw, ck.i0, ck.i1, ck.ext)))
            return rc;
    }
    if (cap) capture(plan, gen_at_entry, fs, args, std::move(chunks[0].steps));
    return ar.finish();
}
