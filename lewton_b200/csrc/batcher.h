// batcher.h -- internals of lwf_batcher (include/lewton_frontend.h) shared by its two halves: frontend.cpp, the
// host entropy decode and the synchronous lwf_batcher_decode, and batcher_submit.cpp, the asynchronous lwf_batcher_submit.
// frontend.cpp needs no CUDA and calls only the synchronous back half, so that it also builds against a stub back half
// (the fuzz harness); whatever submits use beyond that is reached through lwf_batcher::release.
#ifndef LWF_BATCHER_H
#define LWF_BATCHER_H

#include <cstdint>
#include <vector>

#include "../../include/lewton_frontend.h"

namespace lwfb {

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
    std::vector<std::vector<lwb_vq_run>> job_runs;      // LWB_ENTRY_VQ: per-job records before they are packed (kept
    std::vector<std::vector<uint16_t>> job_ents;        // across calls: their capacity is what the next batch needs too)
    uint64_t in_bytes = 0;                              // bytes of the arrays the slice hands to lwb_decode_chains
    uint64_t coeff_total = 0;                           // elements of the slice's coefficient (and dense floor) arena
};

struct JobPlan { uint64_t coeff0, pkt0; uint32_t usable; int32_t head_status; };

struct SubmitRing;      // batcher_submit.cpp: the tickets and device arenas of lwf_batcher_submit

}  // namespace lwfb

struct lwf_batcher {
    lwb_ctx *ctx = nullptr;
    const lwf_headers *hdr = nullptr;
    int threads = 1;
    bool has_floor0 = false;        // the decode can produce dense floor-0 curves: the dense arena is allocated and sent
    bool floor0_records = false;    // lwf_batcher_set_floor0
    int entry = LWB_ENTRY_RESIDUE;  // LWB_ENTRY_VQ: the residue crosses the boundary as VQ records
    // lwf_batcher_decode: slice i decodes into arena[i & 1] while slice i - 1 is being synthesised.
    // lwf_batcher_submit: the two sets form a ring; a submit decodes into the set the submit two back read.
    lwfb::BatchArena arena[2];
    double t_entropy = 0, t_synth = 0;
    uint64_t in_bytes = 0;          // of the last lwf_batcher_decode (all slices) or lwf_batcher_submit
    // Set by the first lwf_batcher_submit: waits for the submits that still read the arena sets (and with destroy, frees
    // the ring and its device arenas).  lwf_batcher_decode and lwf_batcher_destroy call it before they touch the arenas.
    lwfb::SubmitRing *ring = nullptr;
    int (*release)(lwf_batcher *b, bool destroy) = nullptr;
};

namespace lwfb {

double now_s();
// any job without a stream, or with packets but no packet or length array: LWB_ERR_INVALID
int check_jobs(const lwf_stream_job *jobs, size_t n_jobs);
// entropy decode of jobs [j0, j1) into `ar` on the batcher's host threads; fills ar's chains
int batch_entropy(lwf_batcher *b, BatchArena &ar, lwf_stream_job *jobs, size_t j0, size_t j1, std::vector<JobPlan> &plan,
                  std::vector<uint32_t> &decoded, std::vector<int32_t> &dec_status);
// the host-memory batch of arena set `ar`
lwb_batch_io batch_io(const lwf_batcher *b, const BatchArena &ar, int out_format, void *pcm);
// job results of chains [j0, j1) of `ar` after their synthesis
void job_results(lwf_stream_job *jobs, size_t j0, size_t j1, const BatchArena &ar, const std::vector<JobPlan> &plan,
                 const std::vector<uint32_t> &decoded, const std::vector<int32_t> &dec_status);

}  // namespace lwfb

#endif
