// readers.cpp -- lwf_readers (include/lewton_frontend.h): many OggStreamReaders advanced by one call.  Each reader keeps
// what lwf_reader keeps on the host (pager, serial, granule position, where its stream's audio starts) and its own stream
// state.  A read de-pages and counts each job's packets on the batcher's thread pool; a skip walks the packets by their
// sample counts on the pool.  Both then run one batch step (submit_step): each job becomes one chain of an internal
// lwf_batcher's submit, so that its entropy decode and synthesis are exactly lwf_batcher_submit's, and each reader is
// committed from its chain's result or, if the chain was not queued, put back as it was.  A seek walks pages on the pool
// and touches host state only.  The header walk, the serial filter, the granule position and skip rules are the single
// reader's own (batcher.h); what is this file's is applying them ahead of the batch, per job, and committing the reader
// state of the packets the batch ran.  A fresh stream state (first stream, chained stream, after a seek) makes
// its first packet return 0 samples, a chained stream's first audio packet is decoded and dropped, and the cut of a
// stream's last packet is made by the stream's output window.
#include <algorithm>
#include <cstring>
#include <new>
#include <thread>
#include <vector>

#include "batcher.h"
#include "lwb_common.h"

using lwfb::Granule;
using lwfb::ogg_clone;
using lwfb::pager_offset;
using lwfb::run_pool;

namespace {

// One distinct (ident, setup) header byte pair: the headers its streams are entropy-decoded with and their lwb_setup,
// registered with the internal batcher once the setup exists.
struct SharedSet {
    std::vector<uint8_t> ident, setup;
    lwf_headers *h = nullptr;
    lwb_setup *su = nullptr;
};

struct Reader {
    lwf_ogg *ogg = nullptr;
    lwf_headers *hdr = nullptr;        // its comments; ident and setup are its SharedSet's (lwfb::headers_sharing)
    size_t set = 0;                    // its SharedSet
    lwb_stream *pwr = nullptr;         // made by the first read of the stream
    uint32_t serial = 0;
    Granule gp;
    bool fresh = true;                 // the stream state is empty: the next packet returns 0 samples
    bool pending_drop = false;         // a chained stream's headers were read: its first audio packet is dropped next
    uint8_t channels = 0, bs0 = 0, bs1 = 0;
    size_t audio_start = 0;            // pager offset of the first page after the stream's headers (where seeks start)
    // While pending_drop after a read job stopped at a chained stream: the reader as the single reader still stands, in
    // the stream before, with its pager where the single reader's next call reads the new stream's ident.  A seek goes
    // back to it; the drop releases it.  (Readers are copied shallowly: which copy owns what is said where they are.)
    Reader *before_chain = nullptr;
};

// One packet of a job's chain and the reader's accounting once it has been returned
struct Pkt {
    size_t off, len;                   // in Job::bytes
    uint32_t samples;                  // what it returns (0 for the dropped packet)
    size_t calls;                      // pager reads up to and including this packet, from the job's start
    Granule gp;
};

struct Job {
    lwf_ogg *snap = nullptr;           // the pager before the job (swapped back into the reader to restore it)
    std::vector<uint8_t> bytes;
    std::vector<Pkt> pkts;
    bool drop_tried = false;           // the reader's pending drop was read (or the pager failed reading it)
    bool dropped = false;              // pkts[0] is a chained stream's dropped packet
    size_t calls = 0;                  // pager reads the de-paging made
    size_t keep_calls = SIZE_MAX;      // fewer of them to keep, even if every packet runs
    int32_t stop = LWB_OK;             // the pager error that ended the job after pkts (LWB_OK: none)
    bool ended = false, chained = false;
    std::vector<uint8_t> chain_ident;  // chained: the new stream's ident packet (already read)
    size_t limit = SIZE_MAX;           // samples the job may write: set when its last packet is truncated
    ~Job() { lwf_ogg_close(snap); }
};

}  // namespace

struct lwf_readers {
    lwb_ctx *ctx = nullptr;
    int threads = 1;
    std::vector<std::unique_ptr<Reader>> readers;
    std::vector<std::unique_ptr<SharedSet>> sets;
    lwf_batcher *batcher = nullptr;    // made with the first device setup
    std::vector<lwb_stream *> retired; // stream states of streams that a chained stream replaced (queued reads may use them)
    double t_paging = 0, t_entropy = 0, t_synth = 0;   // of the last lwf_readers_read or lwf_readers_skip_samples_linear
};

namespace {

bool same(const std::vector<uint8_t> &v, const uint8_t *p, size_t n) { return v.size() == n && (n == 0 || !std::memcmp(v.data(), p, n)); }

// The shared set of these header packets; a new pair is parsed here, the only parse of its setup header (with
// lwf_headers_parse's errors, those of the comment header included)
int find_set(lwf_readers *rs, const lwfb::HeaderPackets &hp, size_t *out)
{
    const lwf_ogg_packet &setup = hp.setup;
    for (size_t k = 0; k < rs->sets.size(); k++)
        if (same(rs->sets[k]->ident, hp.ident.data(), hp.ident.size()) && same(rs->sets[k]->setup, setup.data, setup.len)) {
            *out = k;
            return LWB_OK;
        }
    std::unique_ptr<SharedSet> s(new SharedSet());
    s->ident = hp.ident;
    s->setup.assign(setup.data, setup.data + setup.len);
    const int rc =
        lwf_headers_parse(hp.ident.data(), hp.ident.size(), hp.comment.data(), hp.comment.size(), setup.data, setup.len, &s->h);
    if (rc) return rc;
    rs->sets.push_back(std::move(s));
    *out = rs->sets.size() - 1;
    return LWB_OK;
}

// read_headers, inside_ogg.rs:19-39 (`first`: the ident packet of a chained stream, already read).  The granule
// position is left alone: a chained stream's dropped packet resets it.  The headers and stream state r held are not
// released: the caller, which keeps a copy of r from before, decides what becomes of them.
int read_headers(lwf_readers *rs, Reader &r, const std::vector<uint8_t> *first)
{
    lwfb::HeaderPackets hp;
    if (first) hp.ident = *first;
    int rc = lwfb::read_header_packets(r.ogg, first != nullptr, hp);
    if (rc) return rc;
    size_t set = 0;
    if ((rc = find_set(rs, hp, &set))) return rc;
    // the reader's own headers hold its comments only: an equal (ident, setup) pair parsed before cannot fail, so the
    // comment header is all that can, with the code the whole parse gives
    lwf_headers *h = nullptr;
    if ((rc = lwfb::headers_sharing(rs->sets[set]->h, hp.comment.data(), hp.comment.size(), &h))) return rc;
    lwf_info info;
    lwf_headers_info(h, &info);
    r.hdr = h;
    r.set = set;
    r.pwr = nullptr;
    r.serial = hp.serial;
    r.fresh = true;
    r.pending_drop = first != nullptr;
    r.channels = info.audio_channels;
    r.bs0 = info.blocksize_0;
    r.bs1 = info.blocksize_1;
    r.audio_start = pager_offset(r.ogg);
    return LWB_OK;
}

// Releases what reader state `old` holds and `now` does not: headers, stream state (retired: queued batches may still
// use it), pager and the reader before a chain.
void release_unshared(lwf_readers *rs, Reader &old, const Reader &now)
{
    if (old.hdr && old.hdr != now.hdr) lwf_headers_destroy(old.hdr);
    if (old.pwr && old.pwr != now.pwr) rs->retired.push_back(old.pwr);
    if (old.ogg != now.ogg) lwf_ogg_close(old.ogg);
    if (old.before_chain && old.before_chain != now.before_chain) {
        release_unshared(rs, *old.before_chain, Reader());
        delete old.before_chain;
    }
}

// The reader enters the chained stream whose headers it has read: the stream before is given up
void drop_before_chain(lwf_readers *rs, Reader &r)
{
    if (!r.before_chain) return;
    Reader *b = r.before_chain;
    r.before_chain = nullptr;
    release_unshared(rs, *b, r);
    delete b;
}

// A read job stopped at a chained stream's ident (`calls` pager reads after the job's start): its headers are read now,
// which the single reader does at its next call, and the reader as the single reader stands is kept until the drop.
int read_chained(lwf_readers *rs, Reader &r, const Job &j, size_t calls)
{
    Reader before = r;
    before.before_chain = nullptr;
    if (!(before.ogg = ogg_clone(j.snap))) return LWB_ERR_BUFFER;
    lwf_ogg_packet pk;
    for (size_t k = 0; k < calls; k++) lwf_ogg_next_packet(before.ogg, &pk);
    Reader *b = new (std::nothrow) Reader(before);
    int rc = b ? read_headers(rs, r, &j.chain_ident) : LWB_ERR_BUFFER;
    if (rc) {
        lwf_ogg_close(before.ogg);
        delete b;
        return rc;
    }
    r.before_chain = b;
    return LWB_OK;
}

// The device setup of r's shared set (registered with the internal batcher) and r's stream state, if not made yet
int ensure_device(lwf_readers *rs, Reader &r)
{
    if (r.pwr) return LWB_OK;
    SharedSet &s = *rs->sets[r.set];
    int rc;
    if (!s.su) {
        lwb_setup *su = nullptr;
        if ((rc = lwf_headers_make_setup(s.h, rs->ctx, &su))) return rc;
        if (!rs->batcher && (rc = lwf_batcher_create(rs->ctx, s.h, rs->threads, &rs->batcher))) {
            lwb_setup_destroy(su);
            return rc;
        }
        if ((rc = lwf_batcher_add_headers(rs->batcher, s.h, su))) {
            lwb_setup_destroy(su);
            return rc;
        }
        s.su = su;
    }
    return lwb_stream_open(rs->ctx, s.su, &r.pwr);
}

// De-pages up to max_packets returned packets of reader r into job j and counts the samples each returns, with the
// reader's granule position after each.  The pager advances (j.snap holds it as it was); the rest of the reader is
// left to the commit, which knows which packets the batch ran.
void depage(const lwf_readers *rs, Reader &r, uint32_t max_packets, Job &j)
{
    if (!max_packets) return;
    bool fresh = r.fresh, direct = false;
    Granule gp = r.gp;
    uint64_t sum = 0;
    lwf_ogg_packet pk;
    int rc = LWB_OK;
    auto next = [&]() {
        j.calls++;
        return lwf_ogg_next_packet(r.ogg, &pk);
    };
    auto add = [&](uint32_t samples) {
        j.pkts.push_back(Pkt{j.bytes.size(), pk.len, samples, j.calls, gp});
        j.bytes.insert(j.bytes.end(), pk.data, pk.data + pk.len);
    };
    if (r.pending_drop) {
        // read_next_audio_packet, inside_ogg.rs:118-141: the chained stream's first audio packet is decoded and dropped
        // (a fresh state: it returns nothing), absgp becomes its page's, and the packet after it is returned whatever
        // its serial
        j.drop_tried = true;
        if ((rc = next())) {
            if (rc == LWF_ERR_NO_MORE_PACKETS) j.ended = true;
            else j.stop = rc;
            return;
        }
        gp = Granule{true, pk.absgp_page};
        add(0);
        j.dropped = true;
        fresh = false;
        direct = true;
    }
    const lwf_headers *H = rs->sets[r.set]->h;
    bool truncated = false;
    for (uint32_t returned = 0; returned < max_packets; returned++) {
        rc = direct ? next() : lwfb::next_packet_of(r.ogg, r.serial, &pk, &j.calls);
        if (rc) {
            if (rc == LWF_ERR_NO_MORE_PACKETS) j.ended = true;
            else j.stop = rc;
            break;
        }
        if (!direct && pk.stream_serial != r.serial) {      // a chained stream begins: the commit reads its headers
            j.chained = true;
            j.chain_ident.assign(pk.data, pk.data + pk.len);
            break;
        }
        direct = false;
        if (truncated) {
            // the stream goes on past the packet its end-of-stream page truncated: the job ends at that packet, so that
            // the window cuts only the job's last packet, and the next job reads this one again
            j.keep_calls = j.pkts.back().calls;
            break;
        }
        size_t cnt = 0;
        if (lwf_decoded_sample_count(H, pk.data, pk.len, &cnt)) {
            add(0);                                   // the batch reports its header error; it is consumed
            break;
        }
        if (fresh) cnt = 0;
        const size_t kept = gp.cut(pk, cnt);
        truncated = kept < cnt;
        gp.step(pk, kept);
        fresh = false;
        add((uint32_t)kept);
        sum += kept;
    }
    if (truncated) j.limit = sum;
}

// Moves r's pager back to where it stood `calls` reads after the job's start: the snapshot is swapped in (nothing is
// allocated) and the reads are made again.
void rewind(Reader &r, Job &j, size_t calls)
{
    std::swap(r.ogg, j.snap);
    lwf_ogg_packet pk;
    for (size_t k = 0; k < calls; k++) lwf_ogg_next_packet(r.ogg, &pk);
}

// The job's results and the reader's state from the batch's result for its chain (sj): packets [0, f) ran, and packet
// f, if there is one, failed and is consumed.  Allocates nothing but at a chained stream's headers, whose failure is
// the job's status.
void commit(lwf_readers *rs, Reader &r, Job &j, const lwf_stream_job &sj, lwf_read_job &out)
{
    const size_t n = j.pkts.size(), D = j.dropped ? 1 : 0;
    const bool failed = sj.status != LWB_OK;
    const size_t f = failed ? sj.packets_done : n;
    const size_t keep = failed && f < n ? j.pkts[f].calls : j.keep_calls;
    if (keep < j.calls) rewind(r, j, keep);
    if (f > 0) r.gp = j.pkts[f - 1].gp;
    else if (j.drop_tried) r.gp.has = false;
    // the state the batch left, read from the stream's host flags: a failing packet may also have cleared it
    r.fresh = lwb_stream_state_len(r.pwr) == 0;
    if (j.drop_tried) {
        r.pending_drop = false;
        drop_before_chain(rs, r);
    }
    out.n_packets = (uint32_t)(f > D ? f - D : 0);
    out.n_samples = sj.n_samples;
    out.channels = r.channels;
    out.next_chained = out.ended = 0;
    out.status = failed ? sj.status : j.stop;
    if (out.packet_samples)
        for (uint32_t i = 0; i < out.n_packets; i++) out.packet_samples[i] = j.pkts[D + i].samples;
    if (failed) return;
    out.ended = j.ended;
    if (j.chained) {
        int rc;
        try {
            rc = read_chained(rs, r, j, f ? j.pkts[f - 1].calls : 0);
        } catch (...) {
            rc = LWB_ERR_BUFFER;
        }
        if (rc) out.status = rc;
        else out.next_chained = 1;
    }
    // packet_samples come from the packets' headers, n_samples from the batch; they agree unless a packet's window
    // flags disagree with the block before it in a way the synthesis does not refuse -- then packet_samples cannot
    // slice the PCM, and the job says so
    uint64_t counted = 0;
    for (size_t i = 0; i < f; i++) counted += j.pkts[i].samples;
    if (counted != sj.n_samples && !out.status) out.status = LWB_ERR_MISMATCH;
}

bool planar(int fmt) { return lwb::out_format_of(fmt).planar; }

// The most samples per channel n consecutive packets of reader r's stream can return: n * blocksize_1 / 2, and once
// (blocksize_1 - blocksize_0) / 4 more, which a long block before a short one returns beyond its half.
uint64_t most_samples(const Reader &r, uint32_t n)
{
    const uint64_t n1 = (uint64_t)1 << r.bs1, n0 = (uint64_t)1 << r.bs0;
    return n ? n * (n1 / 2) + (n1 - n0) / 4 : 0;
}

// A planar out_stride too short for n packets of reader r's stream
bool short_stride(int fmt, uint64_t stride, const Reader &r, uint32_t n) { return planar(fmt) && stride < most_samples(r, n); }

// Unknown or repeated reader indices among n entries `reader(k)`
template <class F> bool bad_readers(const lwf_readers *rs, size_t n, F reader)
{
    std::vector<char> seen(rs->readers.size(), 0);
    for (size_t k = 0; k < n; k++) {
        const uint32_t i = reader(k);
        if (i >= rs->readers.size() || seen[i]) return true;
        seen[i] = 1;
    }
    return false;
}

// ensure_device for the readers `reader(k)` of n jobs
template <class F> int ensure_devices(lwf_readers *rs, size_t n, F reader)
{
    int rc = LWB_OK;
    for (size_t k = 0; k < n && !rc; k++) rc = ensure_device(rs, *rs->readers[reader(k)]);
    return rc;
}

// One job's chain in a batch step
struct StepJob {
    Reader *r = nullptr;               // whose stream state runs the chain
    std::vector<const uint8_t *> packets;
    std::vector<size_t> lengths;
    uint64_t out_offset = 0, out_stride = 0;
    size_t limit = SIZE_MAX;           // the samples the job may write, if its stream's window cuts its last packet
    bool reset = false;                // the chain runs on a reset stream state
    lwfb::StreamFlags flags{false, 0}; // reset: the stream state's flags before it
};

// The batch step of a read or a skip, after its pass on the pool.  `chain(k, c)` gives job k's chain c, whose packet
// bytes the caller keeps; each chain is one job of the internal batcher's lwf_batcher_submit.  A chain on a reset state
// has its stream reset first, and a chain with a limit has its stream's output window set for this submit only.  Then
// settle(k, sj) runs for every job, with its result if it was queued and NULL if not: a job not queued has had its
// stream's flags put back, and the caller puts its reader back.  `rc` is an error already met: nothing is submitted.
// The chains are all made before any stream is reset, so a failure to make one leaves every stream as it was.
template <class Chain, class Settle>
int submit_step(lwf_readers *rs, size_t n, int rc, double paging, int out_format, void *pcm, int pcm_memory, uint64_t *ticket,
                Chain chain, Settle settle)
{
    std::vector<StepJob> c;
    std::vector<lwf_stream_job> sj;
    bool built = false;
    if (!rc) {
        try {
            c.resize(n);
            sj.resize(n);
            for (size_t k = 0; k < n; k++) {
                chain(k, c[k]);
                std::memset(&sj[k], 0, sizeof(sj[k]));
                sj[k].stream = c[k].r->pwr;
                sj[k].n_packets = (uint32_t)c[k].packets.size();
                sj[k].packets = c[k].packets.data();
                sj[k].lengths = c[k].lengths.data();
                sj[k].out_offset = c[k].out_offset;
                sj[k].out_stride = c[k].out_stride;
                sj[k].packets_done = UINT32_MAX;       // still so after the call: the job's batch was not queued
            }
            built = true;
        } catch (...) {
            rc = LWB_ERR_BUFFER;
        }
    }
    uint64_t t = 0;
    if (built) {
        for (size_t k = 0; k < n; k++)
            if (c[k].reset) {
                c[k].flags = lwfb::stream_flags(c[k].r->pwr);
                lwb_stream_reset(c[k].r->pwr);
            }
        for (size_t k = 0; k < n && !rc; k++)
            if (c[k].limit != SIZE_MAX) rc = lwb_stream_set_window(c[k].r->pwr, 0, c[k].limit);
        if (!rc) rc = lwf_batcher_submit(rs->batcher, sj.data(), n, out_format, pcm, pcm_memory, &t);
        for (size_t k = 0; k < n; k++)
            if (c[k].limit != SIZE_MAX) lwb_stream_set_window(c[k].r->pwr, 0, UINT64_MAX);
    }
    for (size_t k = 0; k < n; k++) {
        const bool queued = built && sj[k].packets_done != UINT32_MAX;
        if (built && !queued && c[k].reset) lwfb::set_stream_flags(c[k].r->pwr, c[k].flags);
        settle(k, queued ? &sj[k] : nullptr);
    }
    if (rc) return rc;
    rs->t_paging = paging;
    lwf_batcher_last_timing(rs->batcher, &rs->t_entropy, &rs->t_synth);
    *ticket = t;
    return LWB_OK;
}

int read(lwf_readers *rs, lwf_read_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory, uint64_t *ticket)
{
    auto reader = [&](size_t k) { return jobs[k].reader; };
    if (bad_readers(rs, n_jobs, reader)) return LWB_ERR_INVALID;
    for (size_t k = 0; k < n_jobs; k++)
        if (short_stride(out_format, jobs[k].out_stride, *rs->readers[jobs[k].reader], jobs[k].max_packets)) return LWB_ERR_INVALID;
    int rc = ensure_devices(rs, n_jobs, reader);
    if (rc) return rc;
    std::vector<Job> J(n_jobs);
    for (size_t k = 0; k < n_jobs; k++)
        if (!(J[k].snap = ogg_clone(rs->readers[jobs[k].reader]->ogg))) return LWB_ERR_BUFFER;
    // the readers' de-paging and sample counting on the pool
    const double p0 = lwfb::now_s();
    rc = run_pool(rs->threads, n_jobs, [&](size_t k, int) { depage(rs, *rs->readers[jobs[k].reader], jobs[k].max_packets, J[k]); });
    const double paging = lwfb::now_s() - p0;
    auto chain = [&](size_t k, StepJob &c) {
        const Job &j = J[k];
        c.r = rs->readers[jobs[k].reader].get();
        for (const Pkt &p : j.pkts) {
            c.packets.push_back(j.bytes.data() + p.off);
            c.lengths.push_back(p.len);
        }
        c.out_offset = jobs[k].out_offset;
        c.out_stride = jobs[k].out_stride;
        c.limit = j.limit;              // end-of-stream truncation: the job's last packet is cut by its stream's window
    };
    return submit_step(rs, n_jobs, rc, paging, out_format, pcm, pcm_memory, ticket, chain, [&](size_t k, const lwf_stream_job *sj) {
        Reader &r = *rs->readers[jobs[k].reader];
        if (sj) commit(rs, r, J[k], *sj, jobs[k]);
        else std::swap(r.ogg, J[k].snap);                 // the pager as it was
    });
}

int seek(lwf_readers *rs, const uint32_t *readers, const uint64_t *absgps, size_t n, int32_t *status)
{
    if (bad_readers(rs, n, [&](size_t k) { return readers[k]; })) return LWB_ERR_INVALID;
    rs->retired.reserve(rs->retired.size() + n);       // (release_unshared below cannot fail)
    // a reader whose headers a read took ahead of the single reader goes back to the stream the single reader stands in
    for (size_t k = 0; k < n; k++) {
        Reader &r = *rs->readers[readers[k]];
        if (!r.before_chain) continue;
        Reader *b = r.before_chain;
        Reader now = r;
        r = *b;
        delete b;
        now.before_chain = nullptr;
        release_unshared(rs, now, r);
    }
    const int rc = run_pool(rs->threads, n, [&](size_t k, int) {
        Reader &r = *rs->readers[readers[k]];
        status[k] = lwfb::pager_seek(r.ogg, r.serial, absgps[k], r.audio_start);
    });
    if (rc) return rc;
    // cur_absgp = None and a fresh PreviousWindowRight: host flags only (the ctx's state counter is not the pool's to touch)
    for (size_t k = 0; k < n; k++) {
        if (status[k]) continue;
        Reader &r = *rs->readers[readers[k]];
        r.gp.has = false;
        r.fresh = true;
        if (r.pwr) lwb_stream_reset(r.pwr);
    }
    return LWB_OK;
}

// One skip job: the reader as it was, to restore it if the call is refused, and skip_samples_linear's walk over it
struct Skip {
    Reader saved;                      // (its resources stay the reader's; those the walk replaced are released at commit)
    lwf_ogg *snap = nullptr;           // the pager before the walk
    lwfb::SkipWalk walk;
    uint64_t to_skip0 = 0;
    std::vector<uint8_t> last, drop, target, ident;
    lwf_ogg_packet tpk;                // the target's page facts (its data is `target`)
    size_t tcount = 0;                 // the target's samples by its header
    bool found = false;                // the target was read
    bool has_drop = false;             // the walk dropped the first packet of the chained stream it stands in
    bool boundary = false;             // the walk stopped at a chained stream's ident: its headers are read next
    bool ended = false;
    int32_t stop = LWB_OK;             // the error that ended the walk
    size_t kept = 0;                   // the samples the target returns
    ~Skip() { lwf_ogg_close(snap); }
};

// The entropy decode of a chained stream's first audio packet, the part of its decode and drop that can fail on the
// fresh state it is decoded on
int entropy_check(const lwf_headers *h, const lwf_ogg_packet &pk)
{
    lwfb::PacketScratch scratch(h);
    lwf_decoded_packet dp = scratch.packet();
    return lwf_packet_decode(h, pk.data, pk.len, &dp);
}

// skip_samples_linear's walk of one job (inside_ogg.rs:244-283 with read_next_audio_packet, :107-143), on the pool:
// until the target is read, the stream ends, a packet fails or a chained stream begins (its headers are read between
// rounds, off the pool, since they change the shared sets; the next round drops its first packet and walks on)
void skip_walk(const lwf_readers *rs, Reader &r, Skip &s)
{
    s.boundary = false;
    lwf_ogg_packet pk;
    int rc;
    auto end = [&](int code) {
        if (code == LWF_ERR_NO_MORE_PACKETS) s.ended = true;
        else s.stop = code;
    };
    for (;;) {
        const lwf_headers *H = rs->sets[r.set]->h;
        if (r.pending_drop) {
            r.pending_drop = false;
            r.before_chain = nullptr;          // (released at commit: the walk entered the chained stream)
            r.gp.has = false;
            s.has_drop = false;
            if ((rc = lwf_ogg_next_packet(r.ogg, &pk))) return end(rc);
            if ((rc = entropy_check(H, pk))) return end(rc);
            s.drop.assign(pk.data, pk.data + pk.len);
            s.has_drop = true;
            r.gp = Granule{true, pk.absgp_page};
            if ((rc = lwf_ogg_next_packet(r.ogg, &pk))) return end(rc);     // returned whatever its serial
        } else {
            if ((rc = lwfb::next_packet_of(r.ogg, r.serial, &pk, nullptr))) return end(rc);
            if (pk.stream_serial != r.serial) {
                s.boundary = true;
                s.ident.assign(pk.data, pk.data + pk.len);
                return;
            }
        }
        size_t cnt = 0;
        if ((rc = lwf_decoded_sample_count(H, pk.data, pk.len, &cnt))) return end(rc);
        if (s.walk.target(r.gp, pk, cnt)) {
            s.found = true;
            s.target.assign(pk.data, pk.data + pk.len);
            s.tpk = pk;
            s.tpk.data = nullptr;
            s.tcount = cnt;
            return;
        }
        s.last.assign(pk.data, pk.data + pk.len);
    }
}

// Puts reader r back as it was before job s: the pager, and the headers and stream state the walk made released
// (nothing was queued on them)
void restore_skip(Reader &r, Skip &s)
{
    const Reader now = r;
    r = s.saved;
    std::swap(r.ogg, s.snap);
    if (now.hdr != r.hdr) lwf_headers_destroy(now.hdr);
    if (now.pwr && now.pwr != r.pwr) lwb_stream_destroy(now.pwr);
}

// The job's results and reader r's state from the batch's result for its chain
void commit_skip(lwf_readers *rs, Reader &r, Skip &s, const lwf_stream_job &sj, lwf_skip_job &out)
{
    const bool failed = sj.status != LWB_OK;
    r.fresh = lwb_stream_state_len(r.pwr) == 0;         // as the batch left it, a failing packet's clearing included
    out.channels = r.channels;
    out.got_packet = 0;
    out.n_samples = 0;
    out.left_to_skip = s.to_skip0;
    out.status = failed ? sj.status : s.stop;
    if (!failed && s.found) {
        r.gp.step(s.tpk, s.kept);
        out.got_packet = 1;
        out.n_samples = sj.n_samples;
        out.left_to_skip = s.walk.to_skip;
        if (sj.n_samples != s.kept) out.status = LWB_ERR_MISMATCH;
    } else if (!failed && s.ended) {
        out.left_to_skip = s.walk.to_skip;
    }
    release_unshared(rs, s.saved, r);
}

int skip(lwf_readers *rs, lwf_skip_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory, uint64_t *ticket)
{
    auto reader = [&](size_t k) { return jobs[k].reader; };
    if (bad_readers(rs, n_jobs, reader)) return LWB_ERR_INVALID;
    for (size_t k = 0; k < n_jobs; k++) {
        const Reader &r = *rs->readers[jobs[k].reader];
        if (short_stride(out_format, jobs[k].out_stride, r, 1)) return LWB_ERR_INVALID;
        if (jobs[k].out_channels && jobs[k].out_channels < r.channels) return LWB_ERR_INVALID;
    }
    std::vector<Skip> S(n_jobs);
    rs->retired.reserve(rs->retired.size() + 2 * n_jobs);      // (the commits cannot fail)
    for (size_t k = 0; k < n_jobs; k++) {
        Reader &r = *rs->readers[jobs[k].reader];
        if (!(S[k].snap = ogg_clone(r.ogg))) return LWB_ERR_BUFFER;
        S[k].saved = r;
        S[k].walk.to_skip = S[k].to_skip0 = jobs[k].to_skip;
    }
    // From here a refusal puts every reader back.  The walk, in rounds split at chained streams' headers.
    const double p0 = lwfb::now_s();
    std::vector<size_t> todo(n_jobs);
    for (size_t k = 0; k < n_jobs; k++) todo[k] = k;
    int rc = LWB_OK;
    while (!todo.empty() && !rc) {
        rc = run_pool(rs->threads, todo.size(), [&](size_t t, int) { skip_walk(rs, *rs->readers[jobs[todo[t]].reader], S[todo[t]]); });
        // the chained streams' headers, off the pool.  read_headers changes the reader only once nothing can fail, so
        // after an allocation failure every reader is put back as the others are
        std::vector<size_t> again;
        try {
            again.reserve(todo.size());
            for (size_t t = 0; t < todo.size() && !rc; t++) {
                Skip &s = S[todo[t]];
                if (!s.boundary) continue;
                Reader &r = *rs->readers[jobs[todo[t]].reader];
                const Reader before = r;
                const int hrc = read_headers(rs, r, &s.ident);
                if (hrc) {
                    s.stop = hrc;
                    continue;
                }
                if (before.hdr != s.saved.hdr) lwf_headers_destroy(before.hdr);     // a stream the walk passed through
                again.push_back(todo[t]);
            }
        } catch (...) {
            rc = LWB_ERR_BUFFER;
        }
        todo.swap(again);
    }
    const double paging = lwfb::now_s() - p0;
    // the room of a job whose walk entered a chained stream
    for (size_t k = 0; k < n_jobs && !rc; k++) {
        const Reader &r = *rs->readers[jobs[k].reader];
        if (r.hdr == S[k].saved.hdr) continue;
        const uint64_t room = jobs[k].out_channels ? jobs[k].out_channels : S[k].saved.channels, most = most_samples(r, 1);
        if (r.channels > room || (planar(out_format) ? jobs[k].out_stride < most : room * jobs[k].out_stride < r.channels * most))
            rc = LWB_ERR_INVALID;
    }
    if (!rc) rc = ensure_devices(rs, n_jobs, reader);
    // each job's chain: [packet before, target] on a reset state, [dropped packet, target] on the chained stream's
    // fresh state, the target alone on the reader's state, or the dropped packet alone
    auto chain = [&](size_t k, StepJob &c) {
        Skip &s = S[k];
        c.r = rs->readers[jobs[k].reader].get();
        c.reset = s.found && s.walk.have_last;
        auto add = [&](const std::vector<uint8_t> &p) {
            c.packets.push_back(p.data());
            c.lengths.push_back(p.size());
        };
        if (c.reset) add(s.last);
        else if (s.has_drop) add(s.drop);
        if (s.found) {
            add(s.target);
            const size_t expect = c.reset || s.has_drop || !c.r->fresh ? s.tcount : 0;
            s.kept = c.r->gp.cut(s.tpk, expect);
            if (s.kept < expect) c.limit = s.kept;
        }
        c.out_offset = jobs[k].out_offset;
        c.out_stride = jobs[k].out_stride;
    };
    return submit_step(rs, n_jobs, rc, paging, out_format, pcm, pcm_memory, ticket, chain, [&](size_t k, const lwf_stream_job *sj) {
        Reader &r = *rs->readers[jobs[k].reader];
        if (sj) commit_skip(rs, r, S[k], *sj, jobs[k]);
        else restore_skip(r, S[k]);
    });
}

void destroy_reader(Reader &r)
{
    if (r.pwr) lwb_stream_destroy(r.pwr);
    if (r.hdr) lwf_headers_destroy(r.hdr);
    lwf_ogg_close(r.ogg);
    if (r.before_chain) {
        destroy_reader(*r.before_chain);
        delete r.before_chain;
    }
}

}  // namespace

extern "C" int lwf_readers_create(lwb_ctx *ctx, int threads, lwf_readers **out)
{
    if (!ctx || !out) return LWB_ERR_INVALID;
    lwf_readers *rs = new (std::nothrow) lwf_readers();
    if (!rs) return LWB_ERR_BUFFER;
    rs->ctx = ctx;
    if (threads <= 0) threads = (int)std::thread::hardware_concurrency();
    rs->threads = std::max(1, threads);
    *out = rs;
    return LWB_OK;
}

extern "C" void lwf_readers_destroy(lwf_readers *rs)
{
    if (!rs) return;
    lwf_batcher_destroy(rs->batcher);                  // waits for the reads that still use its arenas
    for (auto &r : rs->readers) destroy_reader(*r);
    for (lwb_stream *s : rs->retired) lwb_stream_destroy(s);
    for (auto &s : rs->sets) {
        if (s->su) lwb_setup_destroy(s->su);
        lwf_headers_destroy(s->h);
    }
    delete rs;
}

extern "C" int lwf_readers_add(lwf_readers *rs, const uint8_t *data, size_t len, uint32_t *index)
{
    if (!rs || (!data && len) || !index || rs->readers.size() >= UINT32_MAX) return LWB_ERR_INVALID;
    std::unique_ptr<Reader> r(new (std::nothrow) Reader());
    if (!r) return LWB_ERR_BUFFER;
    int rc = lwf_ogg_open(data, len, &r->ogg);
    if (rc) return rc;
    rc = lwfb::guarded([&]() -> int {
        const int hrc = read_headers(rs, *r, nullptr);
        if (hrc) return hrc;
        rs->readers.push_back(std::move(r));
        *index = (uint32_t)(rs->readers.size() - 1);
        return LWB_OK;
    });
    if (rc) destroy_reader(*r);     // (r is still held: the push_back failed or was not made)
    return rc;
}

extern "C" const lwf_headers *lwf_readers_headers(const lwf_readers *rs, uint32_t index)
{
    return rs && index < rs->readers.size() ? rs->readers[index]->hdr : nullptr;
}

extern "C" int lwf_readers_last_absgp(const lwf_readers *rs, uint32_t index, uint64_t *absgp)
{
    if (!rs || index >= rs->readers.size() || !absgp) return LWB_ERR_INVALID;
    const Reader &r = *rs->readers[index];
    if (!r.gp.has) return 1;
    *absgp = r.gp.absgp;
    return 0;
}

extern "C" void lwf_readers_last_timing(const lwf_readers *rs, double *paging, double *entropy, double *synthesis)
{
    if (!rs) return;
    if (paging) *paging = rs->t_paging;
    if (entropy) *entropy = rs->t_entropy;
    if (synthesis) *synthesis = rs->t_synth;
}

extern "C" uint32_t lwf_readers_setup_count(const lwf_readers *rs) { return rs ? (uint32_t)rs->sets.size() : 0; }

extern "C" int lwf_readers_read(lwf_readers *rs, lwf_read_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory,
                                uint64_t *ticket)
{
    if (!rs || !jobs || !n_jobs || !pcm || !ticket || (pcm_memory != LWB_MEM_HOST && pcm_memory != LWB_MEM_DEVICE) || !lwb::out_format_known(out_format))
        return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return read(rs, jobs, n_jobs, out_format, pcm, pcm_memory, ticket); });
}

extern "C" int lwf_readers_seek_absgp_pg(lwf_readers *rs, const uint32_t *readers, const uint64_t *absgps, size_t n, int32_t *status)
{
    if (!rs || !readers || !absgps || !n || !status) return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return seek(rs, readers, absgps, n, status); });
}

extern "C" int lwf_readers_skip_samples_linear(lwf_readers *rs, lwf_skip_job *jobs, size_t n_jobs, int out_format, void *pcm,
                                               int pcm_memory, uint64_t *ticket)
{
    if (!rs || !jobs || !n_jobs || !pcm || !ticket || (pcm_memory != LWB_MEM_HOST && pcm_memory != LWB_MEM_DEVICE) || !lwb::out_format_known(out_format))
        return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return skip(rs, jobs, n_jobs, out_format, pcm, pcm_memory, ticket); });
}
