// batcher_submit.cpp -- lwf_batcher_submit (include/lewton_frontend.h): the batcher's entropy decode, then ONE
// asynchronous lwb_submit_chains batch, into host or device PCM.  The entropy decode and the batch's arrays are
// frontend.cpp's (batcher.h); this file adds the ring of arena sets, with the ticket of the submit that last read each
// set, and the device copies of the coefficient and dense floor arenas that device-PCM batches read.
#include <new>
#include <stdexcept>
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

struct SubmitRing {
    DeviceBuf coeffs[2], dense[2];  // device copies of arena[i]'s coeffs / dense arenas (device-PCM submits)
    uint64_t ticket[2] = {0, 0};    // of the last submit that read arena set i, until it has been waited for
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
        for (size_t i = 0; i < 2; i++) {
            b->ring->coeffs[i].release(b->ctx);
            b->ring->dense[i].release(b->ctx);
        }
        delete b->ring;
        b->ring = nullptr;
        b->release = nullptr;
    }
    return rc;
}

// Copies the pinned coefficient and dense floor arenas of set i to their device copies, on the context's stream, so that
// a device-memory batch queued behind the copies reads them there.  *queued: whether a copy was queued.
static int upload_inputs(lwf_batcher *b, size_t i, bool *queued)
{
    const BatchArena &ar = b->arena[i];
    SubmitRing &ring = *b->ring;
    const size_t bytes = (size_t)ar.coeff_total * sizeof(float);
    cudaStream_t st = (cudaStream_t)lwb_ctx_cuda_stream(b->ctx);
    int rc;
    if (b->entry != LWB_ENTRY_VQ) {
        if ((rc = ring.coeffs[i].ensure(b->ctx, bytes))) return rc;
        *queued = bytes != 0;
        if ((rc = ring.coeffs[i].upload(ar.coeffs.p, bytes, st))) return rc;
    }
    if (b->has_floor0) {
        if ((rc = ring.dense[i].ensure(b->ctx, bytes))) return rc;
        *queued |= bytes != 0;
        if ((rc = ring.dense[i].upload(ar.dense.p, bytes, st))) return rc;
    }
    return LWB_OK;
}

static int submit(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory, uint64_t *ticket)
{
    if (!b->ring) {
        b->ring = new SubmitRing();
        b->release = release_ring;
    }
    SubmitRing &ring = *b->ring;
    const size_t i = ring.next;
    BatchArena &ar = b->arena[i];
    const double w0 = now_s();
    int rc = wait_set(b, i);
    const double waited = now_s() - w0;
    if (rc) return rc;
    std::vector<JobPlan> plan(n_jobs);
    std::vector<uint32_t> decoded(n_jobs, 0);
    std::vector<int32_t> dec_status(n_jobs, LWB_OK);
    const double e0 = now_s();
    if ((rc = batch_entropy(b, ar, jobs, 0, n_jobs, plan, decoded, dec_status))) return rc;
    const double s0 = now_s();
    bool queued = false;
    lwb_batch_io io = batch_io(b, ar, out_format, pcm);
    if (pcm_memory == LWB_MEM_DEVICE) {
        // floor and VQ arrays stay in the pinned arenas (floor_memory = LWB_MEM_HOST): the library uploads those itself.
        // An LWB_ENTRY_VQ batch has no coefficient arena (its residue is accumulated on the device).
        rc = upload_inputs(b, i, &queued);
        io.memory = LWB_MEM_DEVICE;
        io.coeffs = b->entry == LWB_ENTRY_VQ ? nullptr : (const float *)ring.coeffs[i].p;
        io.dense_floor = b->has_floor0 ? (const float *)ring.dense[i].p : nullptr;
    }
    uint64_t t = 0;
    if (!rc) rc = lwb_submit_chains(b->ctx, ar.chains.data(), ar.chains.size(), &io, &t);
    if (rc) {
        // no ticket covers the uploads of a refused batch: they finish reading the pinned arenas here
        if (queued) cudaStreamSynchronize((cudaStream_t)lwb_ctx_cuda_stream(b->ctx));
        return rc;
    }
    ring.ticket[i] = t;
    ring.next = (i + 1) % 2;
    job_results(jobs, 0, n_jobs, ar, plan, decoded, dec_status);
    b->t_entropy = s0 - e0;
    b->t_synth = waited + (now_s() - s0);
    b->in_bytes = ar.in_bytes;
    *ticket = t;
    return LWB_OK;
}

}  // namespace lwfb

// One lwb_submit_chains per call, so that a refusal leaves everything as it was; consecutive submits overlap.
extern "C" int lwf_batcher_submit(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory,
                                  uint64_t *ticket)
{
    if (!b || (!jobs && n_jobs) || !pcm || !ticket || (pcm_memory != LWB_MEM_HOST && pcm_memory != LWB_MEM_DEVICE) ||
        lwfb::check_jobs(jobs, n_jobs))
        return LWB_ERR_INVALID;
    try {
        return lwfb::submit(b, jobs, n_jobs, out_format, pcm, pcm_memory, ticket);
    } catch (const std::bad_alloc &) {
        return LWB_ERR_BUFFER;
    } catch (const std::length_error &) {
        return LWB_ERR_BUFFER;
    } catch (...) {
        return LWB_ERR_INVALID;
    }
}
