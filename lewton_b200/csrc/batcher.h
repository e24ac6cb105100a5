// batcher.h -- internals of lwf_batcher (include/lewton_frontend.h) shared by its two halves: frontend.cpp, the
// host entropy decode and the synchronous lwf_batcher_decode, and batcher_submit.cpp, the asynchronous lwf_batcher_submit
// and lwf_batcher_add_headers; and the rules of OggStreamReader, which frontend.cpp's lwf_reader and readers.cpp's
// lwf_readers share.
// frontend.cpp needs no CUDA and calls only the synchronous back half, so that it also builds against a stub back half
// (the fuzz harness); whatever submits and header sets use beyond that is reached through the hooks on lwf_batcher
// (release, set_of).
#ifndef LWF_BATCHER_H
#define LWF_BATCHER_H

#include <cstdint>
#include <functional>
#include <memory>
#include <new>
#include <stdexcept>
#include <vector>

#include "../../include/lewton_frontend.h"

namespace lwfb {

// f() behind the C ABI, which nothing may unwind across: allocation failures (bad_alloc, length_error) become
// LWB_ERR_BUFFER, any other exception LWB_ERR_INVALID.
template <class F> int guarded(F &&f)
{
    try {
        return f();
    } catch (const std::bad_alloc &) {
        return LWB_ERR_BUFFER;
    } catch (const std::length_error &) {
        return LWB_ERR_BUFFER;
    } catch (...) {
        return LWB_ERR_INVALID;
    }
}

struct PinnedBuf {
    void *p = nullptr;
    size_t cap = 0;
    bool ensure(size_t bytes)
    {
        if (bytes <= cap) return true;
        if (p) lwb_host_free(p);
        cap = bytes + bytes / 4 + 4096;
        p = lwb_host_alloc(cap);
        if (!p) cap = 0;
        return p != nullptr;
    }
    ~PinnedBuf() { if (p) lwb_host_free(p); }
};

struct BatchArena {
    PinnedBuf coeffs, dense, kinds, ys, vqrun, vqent, vqroff, vqeoff;
    std::vector<uint8_t> modes, prevs, nexts;
    std::vector<lwb_chain> chains;
    std::vector<size_t> job;                            // the index in the caller's job array of each chain
    std::vector<std::vector<lwb_vq_run>> job_runs;      // LWB_ENTRY_VQ: per-chain records before they are packed (kept
    std::vector<std::vector<uint16_t>> job_ents;        // across calls: their capacity is what the next batch needs too)
    uint64_t in_bytes = 0;                              // bytes of the arrays the batch hands to lwb_decode_chains
    uint64_t coeff_total = 0;                           // elements of the batch's coefficient (and dense floor) arena
};

// The streams of one group share a channel count and a blocksize pair, and go to the synthesis as one batch: the
// library takes residue batches of one channel count only, and a batch of one blocksize pair runs whole on the fused
// kernel of that shape (k_long, the mixed schedule, k_mid) instead of falling to k_chain rounds.
struct Group {
    uint8_t channels = 0, bs0 = 0, bs1 = 0;
    bool has_floor0 = false;        // a header set of the group can produce dense floor-0 curves: the dense arena is sent
    // lwf_batcher_decode: slice i decodes into arena[i & 1] while slice i - 1 is being synthesised.
    // lwf_batcher_submit: the two sets form a ring; a submit decodes into the set the submit two back read.
    BatchArena arena[2];
};

// A set of headers and the setup whose streams it decodes; set 0 is lwf_batcher_create's, for the streams of every
// setup not registered with lwf_batcher_add_headers (its setup is NULL).
struct HeaderSet {
    const lwf_headers *h = nullptr;
    const lwb_setup *setup = nullptr;
    size_t group = 0;
};

struct JobPlan { uint64_t coeff0, pkt0; uint32_t usable; int32_t head_status; size_t set, slot; };

struct SubmitRing;      // batcher_submit.cpp: the tickets and device arenas of lwf_batcher_submit

}  // namespace lwfb

struct lwf_batcher {
    lwb_ctx *ctx = nullptr;
    int threads = 1;
    bool floor0_records = false;    // lwf_batcher_set_floor0
    int entry = LWB_ENTRY_RESIDUE;  // LWB_ENTRY_VQ: the residue crosses the boundary as VQ records
    std::vector<lwfb::HeaderSet> sets;
    std::vector<std::unique_ptr<lwfb::Group>> groups;   // (not moved when a group is added: submits may read their arenas)
    double t_entropy = 0, t_synth = 0;
    uint64_t in_bytes = 0;          // of the last lwf_batcher_decode (all slices) or lwf_batcher_submit (all groups)
    // Set by the first lwf_batcher_submit: waits for the submits that still read the arena sets (and with destroy, frees
    // the ring and its device arenas).  lwf_batcher_decode and lwf_batcher_destroy call it before they touch the arenas.
    lwfb::SubmitRing *ring = nullptr;
    int (*release)(lwf_batcher *b, bool destroy) = nullptr;
    // Set by the first lwf_batcher_add_headers: the header set of the jobs of stream s.  Without it every job has set 0.
    size_t (*set_of)(const lwf_batcher *b, const lwb_stream *s) = nullptr;
};

namespace lwfb {

double now_s();
// The batcher's host thread pool: item(k, w) once for every k in [0, n), on the calling thread (w = 0) and on up to
// min(threads, n) - 1 more (w = 1, 2, ...: a worker's items run one after another), all joined before it returns.  A
// thread that cannot be started leaves its items to the others.  An item that throws ends its worker, whose remaining
// items the others take; the pool then returns LWB_ERR_BUFFER, else LWB_OK.
int run_pool(int threads, size_t n, const std::function<void(size_t k, int w)> &item);
// The buffers one audio packet of a stream decodes into, sized from the stream's headers (floor kinds [C], floor-1 posts
// [C * LWB_MAX_POSTS], dense floor and residue [C * blocksize_1 / 2]), and an lwf_decoded_packet pointing at them
struct PacketScratch {
    std::vector<uint8_t> kinds;
    std::vector<uint32_t> ys;
    std::vector<float> dense, residue;
    PacketScratch() = default;
    explicit PacketScratch(const lwf_headers *h);
    lwf_decoded_packet packet();
};
// An independent copy of a pager's position and buffered packets (nullptr without memory)
lwf_ogg *ogg_clone(const lwf_ogg *o);
// Headers with the comments of `comment` (a comment header packet; lwf_headers_parse's errors for it) that share the
// ident header, codebooks, floors, residues, mappings and modes of `shared`, which must outlive them.  What
// lwf_headers_info, the packet decode and lwf_headers_make_setup give for them is what they give for `shared`.
int headers_sharing(const lwf_headers *shared, const uint8_t *comment, size_t comment_len, lwf_headers **out);

// OggStreamReader's granule position (inside_ogg.rs:219-227): absgp after the packets returned so far, if known.
struct Granule {
    bool has = false;
    uint64_t absgp = 0;
    // of the n samples packet pk decodes to, those it returns: a stream's last packet is cut to its page's granule
    // position (inside_ogg.rs:219-222)
    size_t cut(const lwf_ogg_packet &pk, size_t n) const;
    // after pk returned n samples: the page's granule position at its last packet, else n further on if known (:223-227)
    void step(const lwf_ogg_packet &pk, size_t n);
};

// skip_samples_linear's walk (inside_ogg.rs:244-283) over packets measured by their sample counts only
struct SkipWalk {
    size_t to_skip = 0;
    bool have_last = false;            // last_pck: a packet was measured and passed over before the current one
    // Feeds the next packet pk, whose header says it decodes to n samples.  True: pk is the target (to_skip < its
    // samples after the end-of-stream cut; gp is left for its decode).  False: pk is passed over -- to_skip and gp's
    // absgp (if known, whatever the page, :275-277) go past its samples, and it becomes last_pck.  A stream's last
    // packet, if gp is known, clears last_pck first (:258-262).
    bool target(Granule &gp, const lwf_ogg_packet &pk, size_t n);
};

// The pager's byte offset: where its next page begins
size_t pager_offset(const lwf_ogg *o);
// seek_absgp_pg's page walk (inside_ogg.rs:307-313): the pager moves to the start of the last page of logical stream
// `serial`, at or after byte `from`, whose granule position is <= absgp (its first page if none is).  LWF_ERR_OGG, and
// the pager unchanged, for a bad page on the way or no page of the stream.
int pager_seek(lwf_ogg *o, uint32_t serial, uint64_t absgp, size_t from);

// The header packets of a logical stream, as read_headers (inside_ogg.rs:19-39) gathers them
struct HeaderPackets {
    std::vector<uint8_t> ident, comment;
    lwf_ogg_packet setup;              // a pager packet: valid until the pager's next read
    uint32_t serial = 0;               // the stream's serial, to be adopted
};
// Reads the ident (unless `chained`: a chained stream's, already read into hp.ident), comment and setup packets from o.
// At the start of the data packets of other serials are skipped until those of the ident packet's stream arrive; in
// front of a chained stream the next two packets are taken whatever their serial, and the setup packet's serial is
// adopted (:124-137).  The end of the data is LWF_ERR_OGG.
int read_header_packets(lwf_ogg *o, bool chained, HeaderPackets &hp);
// The serial filter of read_next_audio_packet (inside_ogg.rs:107-117): the next packet of `serial`, or of another
// serial if it begins a logical stream (a chained stream: pk->stream_serial != serial); other packets are skipped.
// *reads (if not NULL) counts the pager reads.
int next_packet_of(lwf_ogg *o, uint32_t serial, lwf_ogg_packet *pk, size_t *reads);
// any job without a stream, or with packets but no packet or length array: LWB_ERR_INVALID
int check_jobs(const lwf_stream_job *jobs, size_t n_jobs);
// plan[j].set for every job
void assign_sets(const lwf_batcher *b, const lwf_stream_job *jobs, size_t n_jobs, std::vector<JobPlan> &plan);
// which groups have dense floor-0 curves, after a header set was added or lwf_batcher_set_floor0
void update_floor0(lwf_batcher *b);
// Entropy decode of jobs list[0 .. n) (plan[j].set assigned) into arena set `set` of their groups, in one parallel pass
// on the batcher's host threads; fills the arenas' chains, each group's in list order.  *used: the groups with jobs in
// the list, ascending, or group 0 alone if the list is empty.
int batch_entropy(lwf_batcher *b, size_t set, lwf_stream_job *jobs, const size_t *list, size_t n, std::vector<JobPlan> &plan,
                  std::vector<uint32_t> &decoded, std::vector<int32_t> &dec_status, std::vector<size_t> *used);
// the host-memory batch of group g's arena set `ar`
lwb_batch_io batch_io(const lwf_batcher *b, size_t g, const BatchArena &ar, int out_format, void *pcm);
// job results of the chains of `ar` after their synthesis
void job_results(lwf_stream_job *jobs, const BatchArena &ar, const std::vector<JobPlan> &plan, const std::vector<uint32_t> &decoded,
                 const std::vector<int32_t> &dec_status);

// lwb_api.cu: what the batcher needs to know of lwb_setup and lwb_stream
struct SetupShape { const lwb_ctx *ctx; uint8_t channels, bs0, bs1; };
SetupShape setup_shape(const lwb_setup *su);
const lwb_setup *stream_setup(const lwb_stream *s);
// A stream's PreviousWindowRight flags (host only): read before lwb_stream_reset, and put back to undo it while no
// batch has been queued on the stream since
struct StreamFlags { bool has; uint32_t plen; };
StreamFlags stream_flags(const lwb_stream *s);
void set_stream_flags(lwb_stream *s, StreamFlags f);
// The refusals lwb_submit_chains would make of this batch (out_format, streams, one channel count, a stream in two
// chains, floor kinds, out_stride, VQ offsets, page-locked host memory), made without queuing anything or changing any state.
int check_submit(lwb_ctx *ctx, const lwb_chain *chains, size_t n_chains, const lwb_batch_io *io);

}  // namespace lwfb

#endif
