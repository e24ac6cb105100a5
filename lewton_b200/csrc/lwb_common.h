// lwb_common.h -- structures shared by the host side and the kernels.
//
// HBM layout (all device-resident, owned by the ctx / setup / stream objects):
//   * per setup:   DevSetup (tables for both blocksizes, floor-1 constants, mappings, modes)
//   * per stream:  state[channels][blocksize_1/2] f32 = PreviousWindowRight (audio.rs:847-861),
//                  the un-windowed right part of the previous block; (has, len) tracked on host
//   * per batch:   coeff arena  [packet][channel][n/2] f32   (spectrum or residue)
//                  pcm arena    planar [chain][channel][stride] or interleaved [chain][t][channel]
//                  DevPacket[]  one descriptor per packet (geometry resolved on the host)
#pragma once
#include <stdint.h>

#include "../../include/lewton_b200.h"

#if defined(__CUDACC__)
#define LWB_CHD __host__ __device__ constexpr
#else
#define LWB_CHD constexpr
#endif

namespace lwb {

// The PCM formats (LWB_OUT_*): all that the batch paths, the launchers and the kernels know about one.  A sample kind
// is one conversion from the f32 sample (samples.rs:86-103); kernel_long.cuh maps it to its element type.
enum SampleKind { kSampleF32 = 0, kSampleI16 = 1, kSampleF16 = 2, kSampleI32 = 3, kSampleI24 = 4 };
constexpr SampleKind kSampleKinds[] = {kSampleF32, kSampleI16, kSampleF16, kSampleI32, kSampleI24};
// The element type of the I24 formats: 3 bytes, little-endian two's complement, byte-aligned (kernel_long.cuh stores it)
struct i24 { unsigned char b[3]; };
static_assert(sizeof(i24) == 3, "packed 3-byte samples");
struct OutFormat {
    unsigned esz;             // bytes per element
    bool planar;              // [channel][out_stride] planes, else [t][channel]
    SampleKind kind;
    unsigned align;           // planar rows at element offsets that are multiples of this start 16-byte aligned (f32, i32)
                              // or at least 8-byte aligned (2-byte samples) in a 16-byte aligned arena: fused_layout
};
constexpr int kOutFormatLast = LWB_OUT_I24_INTERLEAVED;
LWB_CHD bool out_format_known(int f)
{
    return f == LWB_OUT_F32_PLANAR || f == LWB_OUT_I16_PLANAR || f == LWB_OUT_F32_INTERLEAVED || f == LWB_OUT_I16_INTERLEAVED ||
           f == LWB_OUT_F16_PLANAR || f == LWB_OUT_F16_INTERLEAVED || f == LWB_OUT_I32_PLANAR || f == LWB_OUT_I32_INTERLEAVED ||
           f == LWB_OUT_I24_PLANAR || f == LWB_OUT_I24_INTERLEAVED;
}
LWB_CHD OutFormat out_format_of(int f)
{
    return f == LWB_OUT_I16_PLANAR        ? OutFormat{2, true, kSampleI16, 4}
           : f == LWB_OUT_F32_INTERLEAVED ? OutFormat{4, false, kSampleF32, 4}
           : f == LWB_OUT_I16_INTERLEAVED ? OutFormat{2, false, kSampleI16, 4}
           : f == LWB_OUT_F16_PLANAR      ? OutFormat{2, true, kSampleF16, 4}
           : f == LWB_OUT_F16_INTERLEAVED ? OutFormat{2, false, kSampleF16, 4}
           : f == LWB_OUT_I32_PLANAR      ? OutFormat{4, true, kSampleI32, 4}
           : f == LWB_OUT_I32_INTERLEAVED ? OutFormat{4, false, kSampleI32, 4}
           : f == LWB_OUT_I24_PLANAR      ? OutFormat{3, true, kSampleI24, 16}     // 16 samples = 48 bytes
           : f == LWB_OUT_I24_INTERLEAVED ? OutFormat{3, false, kSampleI24, 16}
                                          : OutFormat{4, true, kSampleF32, 4};
}

struct DevTables {            // CachedBlocksizeDerived, header_cached.rs:27-31 (device pointers)
    const float *a, *b, *c, *window;
    const uint32_t *bitrev;
    // fast-path twiddle pack for this blocksize (see kernel_long.cuh), or nullptr
    const float *pack;
    int bs;
    int pad;
};

struct DevFloor1 {            // FloorTypeOne (header.rs:415-424), synthesis-relevant fields only
    uint8_t type;             // LWB_FLOOR_TYPE_*
    uint8_t mult;             // floor1_multiplier
    uint8_t nposts;           // floor1_x_list.len()
    uint8_t pad;
    uint16_t x[LWB_MAX_POSTS];       // floor1_x_list (values <= 1<<15)
    uint8_t sorted[LWB_MAX_POSTS];   // floor1_x_list_sorted[i].0
    uint8_t lo[LWB_MAX_POSTS];       // low_neighbor(x_list, i).0   (audio.rs:285-287), i >= 2
    uint8_t hi[LWB_MAX_POSTS];       // high_neighbor(x_list, i).0  (audio.rs:290-292), i >= 2
};

struct DevMapping {           // Mapping (header.rs:384-390) with mux/submap_floors folded
    uint16_t n_coupling;
    uint16_t pad;
    uint8_t mag[LWB_MAX_COUPLING];
    uint8_t ang[LWB_MAX_COUPLING];
    uint8_t floor_of_channel[LWB_MAX_CHANNELS + 1];   // submap_floors[mux[ch]]
    // channels of every submap in ascending order (the order residue type 2 interleaves them in, audio.rs:957-986);
    // filled for setups with <= 8 channels (LWB_ENTRY_VQ)
    uint8_t sub_nch[LWB_MAX_SUBMAPS];
    uint8_t sub_ch[LWB_MAX_SUBMAPS][8];
};

struct DevBook {              // Codebook (header.rs:360-368): the value table of LWB_ENTRY_VQ
    const float *vq;          // [entries][dims], or nullptr
    uint32_t entries;
    uint16_t dims;
    uint16_t pad;
};
constexpr int kMaxResidues = 64;      // header.rs:973 residue count = read_u6 + 1

struct DevFloor0 {            // FloorTypeZero (header.rs:399-407) as lwb_setup_set_floor0 describes it; order 0 = none
    const float *bark_cos_omega[2];   // cached_bark_cos_omega of blocksize_0 / blocksize_1: n/2 floats each
    float max_amp;            // (1 << amplitude_bits) - 1 as f32 (audio.rs:167-169)
    uint8_t order;            // floor0_order, 2..63
    uint8_t amplitude_offset;
    uint8_t pad[2];
};

struct DevSetup {
    DevTables tab[2];
    const DevFloor1 *floors;
    const DevFloor0 *floor0;  // [n_floors], or nullptr: no floor of the setup has a floor-0 description
    const DevMapping *mappings;
    uint8_t channels, bs0, bs1, n_floors;
    uint8_t mode_blockflag[LWB_MAX_MODES];
    uint8_t mode_mapping[LWB_MAX_MODES];
    // LWB_ENTRY_VQ
    const DevBook *books;
    uint32_t n_books, n_residues;
    uint32_t res_psize[kMaxResidues];  // residue_partition_size
    // output mix (lwb_setup_set_output_mix); n_out == 0: none.  Output channel k sums the terms
    // [mix_row[k], mix_row[k + 1]): input channel mix_ch[j] times mix_w[j], in ascending channel order.
    const uint8_t *mix_ch;
    const float *mix_w;
    uint16_t mix_row[9];
    uint8_t n_out;
};

// One packet of a batch; every index/geometry decision is made on the host
// (audio.rs:1056-1073 window geometry, :1083-1154 which branch of the OLA block runs).
struct DevPacket {
    const DevSetup *setup;
    float *state;             // stream state [channels][state_stride]
    uint64_t coeff_off;       // element offset of [channels][n/2] in the coeff arena
    uint64_t x_off;           // element offset of [channels][n] in the IMDCT scratch (generic path)
    uint64_t out_off;         // element offset of this packet's first sample (channel 0) in the pcm arena
    uint64_t out_stride;      // planar: elements between channel planes
    uint64_t pkt_index;       // row in the per-packet floor arenas
    int32_t prev_packet;      // previous packet of the same chain in this launch, or -1: use `state`
    uint32_t state_stride;    // blocksize_1 / 2
    uint16_t n;               // blocksize of this packet
    uint16_t ls, rs, re;      // left_win_start, right_win_start, right_win_end
    uint16_t plen;            // length of the previous right half; 0 = no previous (no output)
    uint16_t prev_rs;         // right_win_start of prev_packet (where its saved half begins)
    uint8_t blockflag;
    uint8_t mapping;
    uint8_t slope_sel;        // which blocksize's window_slope the left window uses
    uint8_t channels;
    uint8_t save_state;       // last packet of its chain in this launch: write x[rs..re) to state
    uint8_t pad[3];
};

}  // namespace lwb
