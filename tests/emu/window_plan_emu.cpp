// window_plan_emu.cpp -- TEST INFRASTRUCTURE: the output-window clip and the PCM copy-back planner of the host-memory
// batch paths (lewton_b200/csrc/pcm_copy_plan.h), run on the host for chains whose streams have windows, so that the
// copies can be checked against the samples the chains write.
#include <cstddef>
#include <cstdint>

#include "../../lewton_b200/csrc/pcm_copy_plan.h"

// Per chain: produced samples n_samples[i] under window (skip_left[i], limit_left[i]); written[i] and skip[i] out.
// copies: [cap][4] = (off, width, pitch, height) in elements.  Returns the number of copies, or -1 if cap is too small.
extern "C" long lwb_emu_window_plan(int planar, size_t n_chains, const uint32_t *channels, const uint64_t *out_offset,
                                    const uint64_t *out_stride, const uint64_t *n_samples, const uint64_t *skip_left,
                                    const uint64_t *limit_left, uint64_t *skip, uint64_t *written, uint64_t max_pitch,
                                    uint64_t *copies, size_t cap)
{
    std::vector<lwb::PcmSpan> spans;
    std::vector<lwb::PcmCopy> plan;
    for (size_t i = 0; i < n_chains; i++) {
        lwb::window_clip(skip_left[i], limit_left[i], n_samples[i], &skip[i], &written[i]);
        lwb::pcm_chain_spans(planar != 0, channels[i], out_offset[i], out_stride[i], written[i], spans);
    }
    lwb::plan_pcm_copies(spans, max_pitch, plan);
    if (plan.size() > cap) return -1;
    for (size_t k = 0; k < plan.size(); k++) {
        copies[4 * k] = plan[k].off;
        copies[4 * k + 1] = plan[k].width;
        copies[4 * k + 2] = plan[k].pitch;
        copies[4 * k + 3] = plan[k].height;
    }
    return (long)plan.size();
}
