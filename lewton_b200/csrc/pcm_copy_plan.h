// pcm_copy_plan.h -- which elements of the PCM arena a batch's chains write, and the copies that move exactly those
// from a device staging buffer laid out like the arena.  Host code without CUDA types, so that
// tests/emu/copy_plan_emu.cpp can run this source on the CPU.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace lwb {

struct PcmSpan { uint64_t off, len; };                  // arena elements [off, off + len)
// `height` rows of `width` elements, row r at off + r * pitch.  height == 1: one plain span (pitch == width).
struct PcmCopy { uint64_t off, width, pitch, height; };

// The write set of one chain (include/lewton_b200.h, lwb_chain): n samples per channel plane at out_offset + c * out_stride,
// or n * C interleaved samples at out_offset.
inline void pcm_chain_spans(bool planar, unsigned C, uint64_t out_offset, uint64_t out_stride, uint64_t n, std::vector<PcmSpan> &spans)
{
    if (!n || !C) return;
    if (!planar) {
        spans.push_back(PcmSpan{out_offset, n * C});
        return;
    }
    for (unsigned c = 0; c < C; c++) spans.push_back(PcmSpan{out_offset + (uint64_t)c * out_stride, n});
}

// An output window (lwb_stream_set_window) with skip_left samples still to drop and limit_left still to write, over a
// chain that produces n per channel: the chain drops its first *skip samples and writes the next *written.
inline void window_clip(uint64_t skip_left, uint64_t limit_left, uint64_t n, uint64_t *skip, uint64_t *written)
{
    *skip = std::min(skip_left, n);
    *written = std::min(limit_left, n - *skip);
}

// Sorts the spans, merges those that touch or overlap, and emits each run of consecutive merged spans of equal width
// and equal pitch as one copy.  max_pitch (elements) bounds the pitch of a copy of more than one row.  `spans` is
// consumed.  A tight batch (chains adjacent, out_stride == n) is one copy; equal-length chains with padded planes
// are one copy of many rows.
inline void plan_pcm_copies(std::vector<PcmSpan> &spans, uint64_t max_pitch, std::vector<PcmCopy> &copies)
{
    copies.clear();
    if (spans.empty()) return;
    auto by_start = [](const PcmSpan &a, const PcmSpan &b) { return a.off < b.off; };
    if (!std::is_sorted(spans.begin(), spans.end(), by_start)) std::sort(spans.begin(), spans.end(), by_start);
    size_t m = 0;
    for (size_t i = 1; i < spans.size(); i++) {
        PcmSpan &last = spans[m];
        if (spans[i].off <= last.off + last.len) last.len = std::max(last.len, spans[i].off + spans[i].len - last.off);
        else spans[++m] = spans[i];
    }
    spans.resize(m + 1);
    for (size_t i = 0; i < spans.size();) {
        PcmCopy cp{spans[i].off, spans[i].len, spans[i].len, 1};
        size_t j = i + 1;
        if (j < spans.size() && spans[j].len == cp.width && spans[j].off - cp.off <= max_pitch) {
            cp.pitch = spans[j].off - cp.off;
            while (j < spans.size() && spans[j].len == cp.width && spans[j].off == cp.off + cp.height * cp.pitch) {
                cp.height++;
                j++;
            }
        }
        copies.push_back(cp);
        i = j;
    }
}

}  // namespace lwb
