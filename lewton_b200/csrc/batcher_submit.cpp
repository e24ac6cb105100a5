// batcher_submit.cpp -- lwf_batcher_submit (include/lewton_frontend.h): the batcher's entropy decode, then one
// asynchronous lwb_submit_chains batch per group of header sets, into host or device PCM; and lwf_batcher_add_headers,
// which registers those header sets.  The entropy decode and the batches' arrays are frontend.cpp's (batcher.h); this
// file adds the ring of arena sets, with the ticket of the submit that last read each set, and the device copies of the
// coefficient and dense floor arenas that device-PCM batches read.
#include <vector>

#include <cuda_runtime.h>

#include "batcher.h"

namespace lwfb {

// A device copy of a pinned arena (lwb_device_alloc on the batcher's context).
struct DeviceBuf {
    void *p = nullptr;
    size_t cap = 0;
    int device = 0;
    int ensure(lwb_ctx *ctx, size_t bytes)
    {
        if (p && bytes <= cap) return LWB_OK;
        release(ctx);                           // (lwb_device_free synchronises the context's stream)
        const size_t want = bytes + bytes / 4 + 4096;
        const int rc = lwb_device_alloc(ctx, want, &p);
        if (rc) {
            p = nullptr;
            return rc;
        }
        cudaGetDevice(&device);                 // lwb_device_alloc made the context's device current
        cap = want;
        return LWB_OK;
    }
    // `bytes` from pinned `src`, queued on `st`: the copy reads `src` when the stream reaches it
    int upload(const void *src, size_t bytes, cudaStream_t st) const
    {
        if (!bytes) return LWB_OK;
        if (cudaSetDevice(device) != cudaSuccess || cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            cudaGetLastError();
            return LWB_ERR_CUDA;
        }
        return LWB_OK;
    }
    void release(lwb_ctx *ctx)
    {
        if (p) lwb_device_free(ctx, p);
        p = nullptr;
        cap = 0;
    }
};

// The device copies of one group's coeffs / dense arenas, per arena set (device-PCM submits)
struct GroupDevice {
    DeviceBuf coeffs[2], dense[2];
};

struct SubmitRing {
    std::vector<GroupDevice> dev;   // per group
    uint64_t ticket[2] = {0, 0};    // of the last batch that read arena set i, until it has been waited for
    size_t next = 0;                // the set the next submit writes
};

// Waits for the submit that last read arena set i, if it has not been waited for yet.
static int wait_set(lwf_batcher *b, size_t i)
{
    const uint64_t t = b->ring->ticket[i];
    if (!t) return LWB_OK;
    b->ring->ticket[i] = 0;         // a batch that failed on the device does not hold the set either
    return lwb_ticket_wait(b->ctx, t);
}

// lwf_batcher::release
static int release_ring(lwf_batcher *b, bool destroy)
{
    int rc = LWB_OK;
    for (size_t i = 0; i < 2; i++) {
        const int r = wait_set(b, i);
        if (!rc) rc = r;
    }
    if (destroy) {
        for (GroupDevice &d : b->ring->dev)
            for (size_t i = 0; i < 2; i++) {
                d.coeffs[i].release(b->ctx);
                d.dense[i].release(b->ctx);
            }
        delete b->ring;
        b->ring = nullptr;
        b->release = nullptr;
    }
    return rc;
}

// The bytes of group g's coefficient (and dense floor) arena in set i
static size_t arena_bytes(const lwf_batcher *b, size_t g, size_t i) { return (size_t)b->groups[g]->arena[i].coeff_total * sizeof(float); }

// Grows the device copies of group g's arenas of set i to what its batch reads.
static int ensure_inputs(lwf_batcher *b, size_t g, size_t i)
{
    GroupDevice &d = b->ring->dev[g];
    const size_t bytes = arena_bytes(b, g, i);
    int rc;
    if (b->entry != LWB_ENTRY_VQ && (rc = d.coeffs[i].ensure(b->ctx, bytes))) return rc;
    if (b->groups[g]->has_floor0 && (rc = d.dense[i].ensure(b->ctx, bytes))) return rc;
    return LWB_OK;
}

// Copies the pinned coefficient and dense floor arenas of group g's set i to their device copies (grown by
// ensure_inputs), on the context's stream, so that a device-memory batch queued behind the copies reads them there.
// *queued: whether a copy was queued.
static int upload_inputs(lwf_batcher *b, size_t g, size_t i, bool *queued)
{
    const BatchArena &ar = b->groups[g]->arena[i];
    GroupDevice &d = b->ring->dev[g];
    const size_t bytes = arena_bytes(b, g, i);
    cudaStream_t st = (cudaStream_t)lwb_ctx_cuda_stream(b->ctx);
    int rc;
    if (b->entry != LWB_ENTRY_VQ) {
        *queued |= bytes != 0;
        if ((rc = d.coeffs[i].upload(ar.coeffs.p, bytes, st))) return rc;
    }
    if (b->groups[g]->has_floor0) {
        *queued |= bytes != 0;
        if ((rc = d.dense[i].upload(ar.dense.p, bytes, st))) return rc;
    }
    return LWB_OK;
}

// The batch of group g's set i
static lwb_batch_io group_io(lwf_batcher *b, size_t g, size_t i, int out_format, void *pcm, int pcm_memory)
{
    lwb_batch_io io = batch_io(b, g, b->groups[g]->arena[i], out_format, pcm);
    if (pcm_memory == LWB_MEM_DEVICE) {
        // floor and VQ arrays stay in the pinned arenas (floor_memory = LWB_MEM_HOST): the library uploads those itself.
        // An LWB_ENTRY_VQ batch has no coefficient arena (its residue is accumulated on the device).
        const GroupDevice &d = b->ring->dev[g];
        io.memory = LWB_MEM_DEVICE;
        io.coeffs = b->entry == LWB_ENTRY_VQ ? nullptr : (const float *)d.coeffs[i].p;
        io.dense_floor = b->groups[g]->has_floor0 ? (const float *)d.dense[i].p : nullptr;
    }
    return io;
}

static int submit(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory, uint64_t *ticket)
{
    if (!b->ring) {
        b->ring = new SubmitRing();
        b->release = release_ring;
    }
    SubmitRing &ring = *b->ring;
    if (ring.dev.size() < b->groups.size()) ring.dev.resize(b->groups.size());
    const size_t i = ring.next;
    const double w0 = now_s();
    int rc = wait_set(b, i);
    const double waited = now_s() - w0;
    if (rc) return rc;
    std::vector<JobPlan> plan(n_jobs);
    std::vector<uint32_t> decoded(n_jobs, 0);
    std::vector<int32_t> dec_status(n_jobs, LWB_OK);
    std::vector<size_t> all(n_jobs), used;
    for (size_t j = 0; j < n_jobs; j++) all[j] = j;
    assign_sets(b, jobs, n_jobs, plan);
    const double e0 = now_s();
    if ((rc = batch_entropy(b, i, jobs, all.data(), n_jobs, plan, decoded, dec_status, &used))) return rc;
    const double s0 = now_s();
    // Several batches: everything that could refuse one of them is checked, and every arena grown, before the first is
    // queued, so that the refusal of a later batch cannot leave the earlier ones queued.  (One batch is refused or
    // queued as a whole by lwb_submit_chains itself.)
    if (used.size() > 1) {
        for (size_t g : used) {
            if (pcm_memory == LWB_MEM_DEVICE && (rc = ensure_inputs(b, g, i))) return rc;
            const BatchArena &ar = b->groups[g]->arena[i];
            const lwb_batch_io io = group_io(b, g, i, out_format, pcm, pcm_memory);
            if ((rc = check_submit(b->ctx, ar.chains.data(), ar.chains.size(), &io))) return rc;
        }
    }
    uint64_t in_bytes = 0, t = 0;
    for (size_t k = 0; k < used.size(); k++) {
        const size_t g = used[k];
        BatchArena &ar = b->groups[g]->arena[i];
        bool queued = false;
        if (pcm_memory == LWB_MEM_DEVICE && !(rc = ensure_inputs(b, g, i))) rc = upload_inputs(b, g, i, &queued);
        const lwb_batch_io io = group_io(b, g, i, out_format, pcm, pcm_memory);
        uint64_t tg = 0;
        if (!rc) rc = lwb_submit_chains(b->ctx, ar.chains.data(), ar.chains.size(), &io, &tg);
        if (rc) {
            // no ticket covers the uploads of a refused batch: they finish reading the pinned arenas here
            if (queued) cudaStreamSynchronize((cudaStream_t)lwb_ctx_cuda_stream(b->ctx));
            if (k) {
                // LWB_ERR_CUDA or LWB_ERR_BUFFER after the batches of used[0 .. k) were queued: they keep the set
                ring.ticket[i] = t;
                ring.next = (i + 1) % 2;
            }
            return rc;
        }
        t = tg;
        job_results(jobs, ar, plan, decoded, dec_status);
        in_bytes += ar.in_bytes;
    }
    // tickets complete in submission order: the last one covers every batch of the submit
    ring.ticket[i] = t;
    ring.next = (i + 1) % 2;
    b->t_entropy = s0 - e0;
    b->t_synth = waited + (now_s() - s0);
    b->in_bytes = in_bytes;
    *ticket = t;
    return LWB_OK;
}

// lwf_batcher::set_of
static size_t set_of_stream(const lwf_batcher *b, const lwb_stream *s)
{
    const lwb_setup *su = stream_setup(s);
    for (size_t k = 1; k < b->sets.size(); k++)
        if (b->sets[k].setup == su) return k;
    return 0;
}

static int add_headers(lwf_batcher *b, const lwf_headers *h, const lwb_setup *setup)
{
    lwf_info info;
    if (lwf_headers_info(h, &info)) return LWB_ERR_INVALID;
    const SetupShape sh = setup_shape(setup);
    if (sh.ctx != b->ctx || sh.channels != info.audio_channels || sh.bs0 != info.blocksize_0 || sh.bs1 != info.blocksize_1)
        return LWB_ERR_INVALID;
    size_t g = 0;
    while (g < b->groups.size() && !(b->groups[g]->channels == sh.channels && b->groups[g]->bs0 == sh.bs0 && b->groups[g]->bs1 == sh.bs1)) g++;
    b->sets.reserve(b->sets.size() + 1);
    if (g == b->groups.size()) {
        std::unique_ptr<Group> grp(new Group());
        grp->channels = sh.channels;
        grp->bs0 = sh.bs0;
        grp->bs1 = sh.bs1;
        b->groups.push_back(std::move(grp));
    }
    b->sets.push_back(HeaderSet{h, setup, g});
    update_floor0(b);
    b->set_of = set_of_stream;
    return LWB_OK;
}

}  // namespace lwfb

// One lwb_submit_chains per group; a refusal leaves everything as it was; consecutive submits overlap.
extern "C" int lwf_batcher_submit(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory,
                                  uint64_t *ticket)
{
    if (!b || (!jobs && n_jobs) || !pcm || !ticket || (pcm_memory != LWB_MEM_HOST && pcm_memory != LWB_MEM_DEVICE) ||
        lwfb::check_jobs(jobs, n_jobs))
        return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return lwfb::submit(b, jobs, n_jobs, out_format, pcm, pcm_memory, ticket); });
}

// The NULL and LWB_ENTRY_VQ checks come before anything reads the setup or the batcher's context.
extern "C" int lwf_batcher_add_headers(lwf_batcher *b, const lwf_headers *h, const lwb_setup *setup)
{
    if (!b || !h || !setup) return LWB_ERR_INVALID;
    if (b->entry == LWB_ENTRY_VQ && !lwf_headers_vq_capable(h)) return LWB_ERR_INVALID;
    for (const lwfb::HeaderSet &s : b->sets)
        if (s.setup == setup) return LWB_ERR_INVALID;
    return lwfb::guarded([&] { return lwfb::add_headers(b, h, setup); });
}
