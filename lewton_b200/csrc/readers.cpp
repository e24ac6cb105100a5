// readers.cpp -- lwf_readers (include/lewton_frontend.h): many OggStreamReaders advanced by one call.  Each reader keeps
// what lwf_reader keeps on the host (pager, serial, granule position) and its own stream state; a call de-pages and
// counts each job's packets on the batcher's thread pool, then hands the packets to an internal lwf_batcher's submit, so
// that their entropy decode and synthesis are exactly lwf_batcher_submit's.  The header walk, the serial filter and the
// granule position rules are the single reader's own (batcher.h); what is this file's is applying them ahead of the
// batch, per job, and committing the reader state of the packets the batch ran.  A fresh stream state (first stream,
// chained stream) makes its first packet return 0 samples, a chained stream's first audio packet is decoded and
// dropped, and the cut of a stream's last packet is made by the stream's output window.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <new>
#include <thread>
#include <vector>

#include "batcher.h"

using lwfb::Granule;
using lwfb::ogg_clone;
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
    double t_paging = 0, t_entropy = 0, t_synth = 0;   // of the last lwf_readers_read
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
// position is left alone: a chained stream's dropped packet resets it.
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
    if (r.hdr) lwf_headers_destroy(r.hdr);
    if (r.pwr) rs->retired.push_back(r.pwr);
    r.hdr = h;
    r.set = set;
    r.pwr = nullptr;
    r.serial = hp.serial;
    r.fresh = true;
    r.pending_drop = first != nullptr;
    r.channels = info.audio_channels;
    r.bs0 = info.blocksize_0;
    r.bs1 = info.blocksize_1;
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
    if (f > 0) {
        r.gp = j.pkts[f - 1].gp;
        r.fresh = false;
    } else if (j.drop_tried) {
        r.gp.has = false;
    }
    if (j.drop_tried) r.pending_drop = false;
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
            rc = read_headers(rs, r, &j.chain_ident);
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

bool planar(int fmt) { return fmt == LWB_OUT_F32_PLANAR || fmt == LWB_OUT_I16_PLANAR || fmt == LWB_OUT_F16_PLANAR; }

// The most samples per channel n consecutive packets of reader r's stream can return: n * blocksize_1 / 2, and once
// (blocksize_1 - blocksize_0) / 4 more, which a long block before a short one returns beyond its half.
uint64_t most_samples(const Reader &r, uint32_t n)
{
    const uint64_t n1 = (uint64_t)1 << r.bs1, n0 = (uint64_t)1 << r.bs0;
    return n ? n * (n1 / 2) + (n1 - n0) / 4 : 0;
}

int read(lwf_readers *rs, lwf_read_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory, uint64_t *ticket)
{
    std::vector<char> seen(rs->readers.size(), 0);
    for (size_t k = 0; k < n_jobs; k++) {
        const lwf_read_job &q = jobs[k];
        if (q.reader >= rs->readers.size() || seen[q.reader]) return LWB_ERR_INVALID;
        seen[q.reader] = 1;
        const Reader &r = *rs->readers[q.reader];
        if (planar(out_format) && q.out_stride < most_samples(r, q.max_packets)) return LWB_ERR_INVALID;
    }
    int rc;
    for (size_t k = 0; k < n_jobs; k++)
        if ((rc = ensure_device(rs, *rs->readers[jobs[k].reader]))) return rc;
    std::vector<Job> J(n_jobs);
    for (size_t k = 0; k < n_jobs; k++)
        if (!(J[k].snap = ogg_clone(rs->readers[jobs[k].reader]->ogg))) return LWB_ERR_BUFFER;
    // the readers' de-paging and sample counting on the pool
    const double p0 = lwfb::now_s();
    std::atomic<size_t> next_job(0);
    std::atomic<int> pool_failed(0);
    run_pool(rs->threads, n_jobs, [&]() {
        try {
            for (size_t k; (k = next_job.fetch_add(1)) < n_jobs;) depage(rs, *rs->readers[jobs[k].reader], jobs[k].max_packets, J[k]);
        } catch (...) {
            pool_failed.store(1);
        }
    });
    const double paging = lwfb::now_s() - p0;
    std::vector<lwf_stream_job> sj(n_jobs);
    for (lwf_stream_job &q : sj) q.packets_done = UINT32_MAX;   // still so after the call: the job's batch was not queued
    std::vector<std::vector<const uint8_t *>> ptrs(n_jobs);
    std::vector<std::vector<size_t>> lens(n_jobs);
    rc = pool_failed.load() ? LWB_ERR_BUFFER : LWB_OK;
    uint64_t t = 0;
    if (!rc) {
        try {
            for (size_t k = 0; k < n_jobs; k++) {
                const Job &j = J[k];
                for (const Pkt &p : j.pkts) {
                    ptrs[k].push_back(j.bytes.data() + p.off);
                    lens[k].push_back(p.len);
                }
                std::memset(&sj[k], 0, sizeof(sj[k]));
                sj[k].stream = rs->readers[jobs[k].reader]->pwr;
                sj[k].n_packets = (uint32_t)j.pkts.size();
                sj[k].packets = ptrs[k].data();
                sj[k].lengths = lens[k].data();
                sj[k].out_offset = jobs[k].out_offset;
                sj[k].out_stride = jobs[k].out_stride;
                sj[k].packets_done = UINT32_MAX;
            }
        } catch (...) {
            rc = LWB_ERR_BUFFER;
        }
    }
    if (!rc) {
        // end-of-stream truncation: the job's last packet is cut by its stream's window, for this batch only
        for (size_t k = 0; k < n_jobs && !rc; k++)
            if (J[k].limit != SIZE_MAX) rc = lwb_stream_set_window(rs->readers[jobs[k].reader]->pwr, 0, J[k].limit);
        if (!rc) rc = lwf_batcher_submit(rs->batcher, sj.data(), n_jobs, out_format, pcm, pcm_memory, &t);
        for (size_t k = 0; k < n_jobs; k++)
            if (J[k].limit != SIZE_MAX) lwb_stream_set_window(rs->readers[jobs[k].reader]->pwr, 0, UINT64_MAX);
    }
    for (size_t k = 0; k < n_jobs; k++) {
        Reader &r = *rs->readers[jobs[k].reader];
        if (sj[k].packets_done == UINT32_MAX) std::swap(r.ogg, J[k].snap);     // not queued: the pager as it was
        else commit(rs, r, J[k], sj[k], jobs[k]);
    }
    if (rc) return rc;
    rs->t_paging = paging;
    lwf_batcher_last_timing(rs->batcher, &rs->t_entropy, &rs->t_synth);
    *ticket = t;
    return LWB_OK;
}

void destroy_reader(Reader &r)
{
    if (r.pwr) lwb_stream_destroy(r.pwr);
    if (r.hdr) lwf_headers_destroy(r.hdr);
    lwf_ogg_close(r.ogg);
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
    if (!rs || !jobs || !n_jobs || !pcm || !ticket || (pcm_memory != LWB_MEM_HOST && pcm_memory != LWB_MEM_DEVICE) || out_format < 0 ||
        out_format > LWB_OUT_F16_INTERLEAVED)
        return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return read(rs, jobs, n_jobs, out_format, pcm, pcm_memory, ticket); });
}
