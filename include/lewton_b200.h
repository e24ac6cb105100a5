/*
 * lewton_b200.h -- C ABI of the H100-native Vorbis packet-synthesis back-end.
 *
 * What it replaces (RustAudio/lewton @ bb2955b): the dense back half of
 *   audio::read_audio_packet_generic            src/audio.rs:988-1157
 * i.e. inverse channel coupling (:991-1002), floor-1 curve synthesis
 * (:391-555) and floor x residue (:1006-1039), imdct::inverse_mdct
 * (src/imdct.rs:291-659), window / overlap-add / PreviousWindowRight
 * (:1056-1154) and Samples::from_floats (src/samples.rs:20-103).  The bit-serial
 * front half (:921-986: mode bits, floor_decode, residue_packet_decode) stays in
 * Rust on the host and hands its dense results across this boundary.
 *
 * Style follows the crate's own C API (src/capi.rs:78-147): opaque pointers,
 * int status, out-parameters, explicit *_destroy.  Nothing unwinds across the
 * boundary.  There is NO CPU fallback: every entry point that computes fails
 * with LWB_ERR_NO_DEVICE / LWB_ERR_CUDA when no sm_90 device is usable.
 *
 * Threading: a ctx is bound to one CUDA device and is not thread-safe (the
 * reference is single-threaded and &mut-exclusive per stream); use one ctx per
 * host thread / per GPU.  Streams of one ctx are independent; packets of one
 * stream must be submitted in order (overlap-add dependency).
 *
 * All arithmetic is IEEE binary32, round-to-nearest, never contracted, in the
 * reference's operation order: f32 PCM is bit-identical to lewton's own output
 * (up to the sign of zero / NaN payload), i16 PCM is bit-identical, f16 PCM is
 * the round-to-nearest-even binary16 of that f32 PCM, i32 and i24 PCM are that
 * f32 PCM scaled, truncated and saturated as lewton's i16 rule does.
 */
#ifndef LEWTON_B200_H
#define LEWTON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: lwb_batch_io::floor_memory, lwb_bind_host_to_device; 3: LWB_ENTRY_VQ.  lwb_submit_chains / lwb_ticket_query /
 * lwb_ticket_wait were added under 3 without a bump: they change no struct and no existing call, so every ABI-3
 * caller keeps working, and the number stays what existing ABI-3 callers (and the project's ABI test) check for.  A
 * caller that needs the asynchronous calls resolves lwb_submit_chains (dlsym) rather than testing the version. */
#define LWB_ABI_VERSION 3
#define LWB_MAX_POSTS 65          /* header.rs:873 floor1_values <= 65 */
#define LWB_MAX_CHANNELS 255      /* audio_channels is a u8, header.rs:190 */
#define LWB_MAX_COUPLING 256      /* header.rs:998-1001 coupling steps = read_u8 + 1 */
#define LWB_MAX_SUBMAPS 16        /* header.rs:994-997 submaps = read_u4 + 1 */
#define LWB_MAX_MODES 64          /* header.rs:1134 mode count = read_u6 + 1 */

/* status codes (0 = ok), cf. audio::AudioReadError (audio.rs:26-41) */
enum {
    LWB_OK = 0,
    LWB_ERR_BAD_FORMAT = 1,   /* AudioReadError::AudioBadFormat (mode index, OLA guard :1107-1111) */
    LWB_ERR_BUFFER = 2,       /* AudioReadError::BufferNotAddressable / output capacity too small */
    LWB_ERR_MISMATCH = 3,     /* where the reference panics: channel-count mismatch (:1086), mag==ang (:783) */
    LWB_ERR_INVALID = 4,      /* NULL / out-of-range argument */
    LWB_ERR_CUDA = 5,         /* a CUDA call failed; see lwb_last_error */
    LWB_ERR_NO_DEVICE = 6     /* no usable sm_90 device: there is no CPU fallback */
};

typedef struct lwb_ctx lwb_ctx;        /* one per GPU: stream, staging, launch state           */
typedef struct lwb_setup lwb_setup;    /* what IdentHeader + SetupHeader give the synthesis half */
typedef struct lwb_stream lwb_stream;  /* PreviousWindowRight (audio.rs:847-861), device-resident */

/* ---- library / context ------------------------------------------------------------------ */
int lwb_abi_version(void);
/* number of CUDA devices visible (0 on a CPU-only host; never fails) */
int lwb_device_count(void);
int lwb_ctx_create(int device_ordinal, lwb_ctx **out);
void lwb_ctx_destroy(lwb_ctx *ctx);
/* block until everything submitted on this ctx has finished (kernels and copies; every ticket completes) */
int lwb_ctx_synchronize(lwb_ctx *ctx);
/* text of the last failure on this ctx (never NULL) */
const char *lwb_last_error(const lwb_ctx *ctx);
/* the cudaStream_t all work of this ctx is launched on (for CUDA-event timing by a harness) */
void *lwb_ctx_cuda_stream(lwb_ctx *ctx);
/* kernels launched by this ctx since creation (bench.py's gpu_launches) */
uint64_t lwb_ctx_launch_count(const lwb_ctx *ctx);
/* The kernels a batch can launch, one id per __global__ function (k_mid's n = 1024 and n = 512 instances share
 * one).  Which of them ran tells which batch path took a batch: every path gives the same bytes. */
enum { LWB_KERNEL_LONG = 0, LWB_KERNEL_LONG_S = 1, LWB_KERNEL_MID = 2, LWB_KERNEL_SHORT = 3, LWB_KERNEL_SHORT_G = 4,
       LWB_KERNEL_ROW_COPY = 5, LWB_KERNEL_CHAIN = 6, LWB_KERNEL_FLOOR1_SEGMENTS = 7, LWB_KERNEL_PROLOGUE_FUSED = 8,
       LWB_KERNEL_PROLOGUE = 9, LWB_KERNEL_IMDCT = 10, LWB_KERNEL_OVERLAP = 11, LWB_KERNEL_SAVE_STATE = 12,
       LWB_KERNEL_FLOOR0_CURVES = 13, LWB_KERNEL_COUNT = 14 };
/* debug: launches of kernel `kernel_id` (LWB_KERNEL_*) by this ctx since creation (0 for an unknown id); the
 * counts of all ids sum to lwb_ctx_launch_count */
uint64_t lwb_ctx_kernel_launches(const lwb_ctx *ctx, int kernel_id);
/* pinned host memory for the host-buffer entry points (optional for lwb_decode_chains, where plain malloc'd memory
 * works, slower; required for a host-memory lwb_submit_chains) */
void *lwb_host_alloc(size_t bytes);
void lwb_host_free(void *p);
/* Multi-GPU hosts: bind the calling thread (and the threads it creates) to the CPUs of the NUMA node GPU
 * `device_ordinal` is attached to and prefer that node's memory, so that pinned buffers allocated afterwards
 * (lwb_host_alloc, staging) are local to the GPU's PCIe root.  Call once per rank / per feeding thread before
 * allocating.  Returns the node, or -1 if unknown (nothing changed).  device_ordinal < 0 restores the default
 * memory policy (the CPU affinity is the caller's to restore).  No reference counterpart: lewton is CPU-only. */
int lwb_bind_host_to_device(int device_ordinal);
/* device memory helpers for the *_DEVICE memory space (harnesses without their own allocator) */
int lwb_device_alloc(lwb_ctx *ctx, size_t bytes, void **out);
void lwb_device_free(lwb_ctx *ctx, void *p);
int lwb_memcpy_h2d(lwb_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int lwb_memcpy_d2h(lwb_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);

/* ---- blocksize-derived tables: header_cached.rs:33-110 ----------------------------------- */
/* CachedBlocksizeDerived::from_blocksize, evaluated on the host with libm sinf/cosf in the
 * reference's f32 expression order.  a,b: n/2 floats; c: n/4; window: n/2; bitrev: n/8. */
int lwb_tables_generate(int blocksize_log2, float *a, float *b, float *c, float *window,
                        uint32_t *bitrev);

/* ---- setup: the header-derived constants the synthesis half reads ------------------------- */
typedef struct lwb_tables_ref {      /* IdentHeader.cached_bs_derived[i], header.rs:210           */
    const float *a, *b, *c;          /* TwiddleFactors, header_cached.rs:20-24                     */
    const float *window;             /* window_slope                                               */
    /* compute_bitreverse(bs) (header_cached.rs:101-110), the only table the crate makes: the fused kernels build that
     * permutation into their index maps, so lwb_setup_create refuses any other with LWB_ERR_INVALID (no setup is
     * created; lwb_last_error says which table).  a, b, c and window may hold any values. */
    const uint32_t *bitrev;
} lwb_tables_ref;

enum { LWB_FLOOR_TYPE_ZERO = 0, LWB_FLOOR_TYPE_ONE = 1 };
typedef struct lwb_floor_desc {      /* header::Floor, header.rs:399-424                           */
    uint8_t floor_type;              /* type 0: dense curves, or records (lwb_setup_set_floor0)    */
    uint8_t floor1_multiplier;       /* 1..4                                                       */
    uint8_t floor1_values;           /* floor1_x_list.len(), 2..65                                 */
    uint8_t reserved;
    uint32_t floor1_x_list[LWB_MAX_POSTS];   /* unsorted, as parsed (header.rs:878-884)            */
} lwb_floor_desc;

typedef struct lwb_mapping_desc {    /* header::Mapping, header.rs:384-390                         */
    uint16_t coupling_steps;
    uint8_t submaps;
    uint8_t reserved;
    uint8_t magnitudes[LWB_MAX_COUPLING];
    uint8_t angles[LWB_MAX_COUPLING];
    uint8_t mux[LWB_MAX_CHANNELS + 1];       /* mapping_mux[channel] -> submap                     */
    uint8_t submap_floors[LWB_MAX_SUBMAPS];  /* submap -> floor index                              */
} lwb_mapping_desc;

typedef struct lwb_mode_desc {       /* header::ModeInfo, header.rs:393-396                        */
    uint8_t blockflag;
    uint8_t mapping;
} lwb_mode_desc;

/* Codebook value tables and residue shapes (only for LWB_ENTRY_VQ batches; leave the counts 0 otherwise). */
typedef struct lwb_codebook_desc {   /* header::Codebook, header.rs:360-368                            */
    uint16_t dimensions;             /* codebook_dimensions                                            */
    uint16_t reserved;
    uint32_t entries;                /* codebook_entries                                               */
    const float *vq;                 /* codebook_vq_lookup_vec: [entries][dimensions]; NULL = no value mapping */
} lwb_codebook_desc;
typedef struct lwb_residue_desc {    /* header::Residue, header.rs:370-379                             */
    uint8_t residue_type;            /* 0, 1, 2                                                        */
    uint8_t reserved[3];
    uint32_t partition_size;         /* residue_partition_size                                         */
} lwb_residue_desc;

typedef struct lwb_setup_desc {
    uint8_t audio_channels;          /* IdentHeader.audio_channels                                 */
    uint8_t blocksize_0, blocksize_1;/* log2, 6..13, blocksize_0 <= blocksize_1 (header.rs:239-243)    */
    uint8_t reserved;
    /* optional: the crate's own tables (so results cannot depend on the libm behind them);
     * a NULL `a` means "generate with lwb_tables_generate" */
    lwb_tables_ref tables[2];
    uint32_t n_floors;
    const lwb_floor_desc *floors;
    uint32_t n_mappings;
    const lwb_mapping_desc *mappings;
    uint32_t n_modes;
    const lwb_mode_desc *modes;
    /* LWB_ENTRY_VQ only (ABI 3; zero / NULL otherwise) */
    uint32_t n_codebooks;
    const lwb_codebook_desc *codebooks;
    uint32_t n_residues;
    const lwb_residue_desc *residues;
} lwb_setup_desc;

int lwb_setup_create(lwb_ctx *ctx, const lwb_setup_desc *desc, lwb_setup **out);
void lwb_setup_destroy(lwb_setup *setup);

/* Floor type 0 on the device (added under ABI 3: no struct above changes).  A type-0 floor described here can be sent
 * as LWB_FLOOR_ZERO records instead of dense LWB_FLOOR_DENSE curves; the device then computes the curve
 * (floor_zero_compute_curve, audio.rs:160-212) bit for bit.  NULL bark_cos_omega tables are generated on the host with
 * libm cosf / atanf in the order of header_cached.rs:129-158. */
typedef struct lwb_floor0_desc {     /* header::FloorTypeZero, header.rs:399-407                       */
    uint8_t order;                   /* floor0_order, 2..63 (a record holds at most 63 coefficients)    */
    uint8_t amplitude_bits;          /* 1..64                                                          */
    uint8_t amplitude_offset;
    uint8_t reserved;
    uint16_t rate;                   /* floor0_rate                                                    */
    uint16_t bark_map_size;          /* floor0_bark_map_size                                           */
    const float *bark_cos_omega[2];  /* cached_bark_cos_omega for blocksize_0 / blocksize_1 (n/2 floats each), or NULL */
} lwb_floor0_desc;
/* Describes floor `floor_index` (of type LWB_FLOOR_TYPE_ZERO in the setup's lwb_floor_desc) for LWB_FLOOR_ZERO rows.
 * Call it before the setup's first batch.  LWB_ERR_INVALID for a bad index, a floor of type 1 or a field out of range. */
int lwb_setup_set_floor0(lwb_setup *setup, uint32_t floor_index, const lwb_floor0_desc *desc);

/* Output channel mix (added under ABI 3: no struct above changes).  Every chain of a stream opened on the setup then
 * writes K = n_out output channels instead of the stream's C = audio_channels (Vorbis I section 4.3.9 order):
 * reordering (e.g. to the WAV / WAVEFORMATEXTENSIBLE order), selection, mono / stereo downmix and duplication.
 *   matrix: [n_out][C] row-major f32, 1 <= n_out <= 8; n_out == 0 with matrix == NULL clears the mix.
 *   Refused with LWB_ERR_INVALID, nothing changed: a NULL setup, n_out out of range, a non-finite coefficient, a call
 *   after any stream has been opened on the setup.
 * Value, bit for bit and without FMA: with x_c[t] the f32 sample the F32 formats write without a mix, y_k[t] is the
 * left-to-right f32 sum, over ascending c with M[k][c] != 0, of the rounded products M[k][c] * x_c[t] (the first term
 * is not added to a zero; a row without a nonzero coefficient gives +0.0f); y is then converted like any f32 sample.
 * A row with a single 1.0f copies its channel exactly, so permutations and selections are bit-exact.
 * Layout: planar, n_samples per plane at out_offset + k * out_stride; interleaved, n_samples * K elements at out_offset;
 * lwb_decode_packet / lwb_decode_spectrum write [K][capacity] or [capacity][K].  Nothing else changes: n_samples,
 * packets_done, status and the stream state (still C channels) are what the same batch gives without a mix.  Setups with
 * and without a mix may share a batch; such a batch runs on the chain kernel or the four-kernel path. */
int lwb_setup_set_output_mix(lwb_setup *setup, uint32_t n_out, const float *matrix);
/* K: n_out of the setup's mix, or audio_channels without one (0 for a NULL setup) */
uint32_t lwb_setup_output_channels(const lwb_setup *setup);

/* ---- stream state: PreviousWindowRight, audio.rs:847-861 ---------------------------------- */
int lwb_stream_open(lwb_ctx *ctx, const lwb_setup *setup, lwb_stream **out);
void lwb_stream_destroy(lwb_stream *s);
/* PreviousWindowRight::new(): the next packet yields 0 samples (audio.rs:1140-1151) */
int lwb_stream_reset(lwb_stream *s);
/* PreviousWindowRight::is_empty() */
int lwb_stream_is_empty(const lwb_stream *s);
/* #[derive(Clone)]: an independent copy of the state */
int lwb_stream_clone(const lwb_stream *s, lwb_stream **out);
/* Output window of a stream (added under ABI 3: no struct or existing call changes).  Of the samples its packets produce
 * from the next queued packet on, the first `skip` per channel are not written, the next `limit` are, and none after
 * that (limit = UINT64_MAX: no end).  Decoding and the stream state are unchanged: every packet still decodes and
 * advances PreviousWindowRight exactly as without a window.  skip = 0, limit = UINT64_MAX is the default and is what
 * every existing caller gets.  It is how a caller gets lewton's sample count at the end of a stream (the last packet
 * truncated to the page's granule position, inside_ogg.rs:219-222) and sample-exact starts after a seek, without a pass
 * of its own over the PCM.
 *   Placement: written sample j of a chain (0-based among the written ones) goes to out_offset + k * out_stride + j
 *     (planar) or to out_offset + j * K + k (interleaved), K = lwb_setup_output_channels.  lwb_chain.n_samples is the
 *     number of samples written, and the out_stride and range checks of a batch use that number.  Nothing outside the
 *     written set changes, in either memory space.
 *   When it moves: the counters advance where the stream state's (has, len) does -- when a batch is queued, at call
 *     time, for lwb_decode_chains, lwb_submit_chains and lwb_plan_execute alike -- so consecutive submits, and windows
 *     that span several batches, behave as one stream.  A refused batch moves no counter; after LWB_ERR_CUDA the counters
 *     are handled like the states: not committed on the host.
 *   lwb_stream_reset leaves the window alone (a seek is a reset followed by lwb_stream_set_window); lwb_stream_clone
 *   copies it; lwb_streams_save / lwb_streams_load do not carry it (the slot format is fixed).  Setting a window makes
 *   prepared batches that hold the stream plan again; lwb_plan_execute replays a prepared batch only while none of its
 *   streams has a window other than the default, so a stream whose limit has run out to 0 keeps its batches planning
 *   every execution until lwb_stream_set_window(s, 0, UINT64_MAX).  lwb_decode_packet and lwb_decode_spectrum honour
 *   the window too.
 *   Memory: a clipped chain decodes its full output into scratch first.  Host-memory batches stage it beside their PCM;
 *   device-memory batches keep it in a device buffer of the context that grows to the largest batch's clipped output
 *   (all chains of a batch clipped: about the size of its PCM) and is freed with the context.
 *   A NULL stream is refused with LWB_ERR_INVALID. */
int lwb_stream_set_window(lwb_stream *s, uint64_t skip, uint64_t limit);
/* what is left of the window: skip still to drop, limit still to write (UINT64_MAX: no end); either pointer may be NULL */
int lwb_stream_window(const lwb_stream *s, uint64_t *skip_left, uint64_t *limit_left);
/* debug / checkpoint: per-channel length of the saved right half (0 if empty), and its data */
uint32_t lwb_stream_state_len(const lwb_stream *s);
int lwb_stream_export_state(lwb_stream *s, float *out /* [channels][len] */);
int lwb_stream_import_state(lwb_stream *s, const float *data /* [channels][len] */, uint32_t len);

/* Many streams' states in one call (added under ABI 3: no struct above changes).  A decode server checkpoints thousands
 * of streams per step, restores them after LWB_ERR_CUDA, and moves them to another context or GPU; one export / import
 * per stream costs a synchronisation each.  Slot i names a stream and where its state lies in `buf`.
 *   Values: slot i of a save holds exactly what lwb_stream_export_state gives for its stream: [channels][len] f32 rows,
 *     contiguous at buf + offset.  Loading those values gives a stream that decodes every later packet exactly as the
 *     saved one would (f32 bit for bit, i16 and f16 exactly, on every batch path).  has = 1 with len = 0 is a state (what
 *     lwb_stream_import_state(s, NULL, 0) makes) and round-trips; has = 0 is PreviousWindowRight::new().
 *   Ordering: both calls are stream-ordered on lwb_ctx_cuda_stream(ctx), like lwb_submit_chains, and draw *ticket from the
 *     same sequence.  A save queued after a submit sees the states that submit leaves; a load queued before a submit is
 *     what that submit starts from.  The host (has, len) of a stream moves at call time, as a submit's does: a save writes
 *     the slots' len and has before it returns, a load sets the streams' (has, len) and makes prepared batches
 *     (lwb_plan_execute) plan again.  A save's rows are in `buf` once its ticket completes; a load reads `buf` until its
 *     ticket completes.
 *   Memory: LWB_MEM_DEVICE: `buf` is device memory of ctx's device, used in place (any alignment; 16-byte aligned rows of
 *     a multiple of 4 floats move as float4s).  LWB_MEM_HOST: `buf` must be page-locked at the first and the last byte
 *     the slots touch, as for a host-memory lwb_submit_chains; pageable memory is refused.  A host-memory call is staged
 *     in the context's device arenas: a load uploads the extent of its slots (lowest offset to highest end, gaps
 *     included) in one copy, a save downloads exactly the slots' rows, in one copy when they are adjacent.
 *   Refusals, before anything changes (no stream state, no slot, no buffer, no ticket):
 *     LWB_ERR_INVALID: a NULL ctx, buf or ticket (slots may be NULL when n == 0), a bad memory space, a slot without a
 *       stream or with a stream of another context, a stream in two slots, a load slot with has == 0 and len != 0,
 *       host memory that is not page-locked;
 *     LWB_ERR_BUFFER: a load slot's len above blocksize_1 / 2 of its stream's setup, or a slot whose range
 *       (offset + channels * len elements, in bytes) would wrap past 2^64.
 *   Across contexts: a buffer saved by one context may be loaded by another, on the same or another device (moving the
 *     bytes between devices is the caller's).  Nothing orders the two contexts' streams: the caller waits on the save's
 *     ticket before it queues the load.  The load reads `channels` rows of len floats per slot, channels of the loading
 *     stream's setup, so the two streams need equal channel counts; their setups need only len <= blocksize_1 / 2 of the
 *     loading one, the rule of lwb_stream_import_state. */
typedef struct lwb_state_slot {
    lwb_stream *stream;
    uint64_t offset;     /* element offset of this stream's [channels][len] f32 rows in `buf`                     */
    uint32_t len;        /* save: written (lwb_stream_state_len); load: read, <= blocksize_1 / 2                  */
    uint8_t has;         /* save: written (!lwb_stream_is_empty); load: read (0 = PreviousWindowRight::new())     */
    uint8_t reserved[3];
} lwb_state_slot;
int lwb_streams_save(lwb_ctx *ctx, lwb_state_slot *slots, size_t n, int memory, float *buf, uint64_t *ticket);
int lwb_streams_load(lwb_ctx *ctx, const lwb_state_slot *slots, size_t n, int memory, const float *buf, uint64_t *ticket);

/* audio::get_decoded_sample_count (audio.rs:874-909) for an already-parsed packet header:
 * right_win_start - left_win_start; does not look at the stream state. */
int lwb_decoded_sample_count(const lwb_setup *setup, uint8_t mode_number, int prev_window_flag,
                             int next_window_flag, uint32_t *n_samples);

/* ---- one packet (mirrors read_audio_packet_generic's back half) --------------------------- */
enum { LWB_FLOOR_UNUSED = 0,   /* DecodedFloor::Unused  -> zero curve (audio.rs:1021-1024)        */
       LWB_FLOOR_ONE = 1,      /* DecodedFloor::TypeOne -> raw floor1_y from floor_one_decode      */
       LWB_FLOOR_DENSE = 2,    /* DecodedFloor::TypeZero -> curve computed by the host (n/2 f32)   */
       LWB_FLOOR_ZERO = 3 };   /* DecodedFloor::TypeZero -> a floor-0 record in the floor1_y row:  *
                                * words 0-1 the amplitude (u64, low word first), words 2 .. 2 + order *
                                * - 1 the coefficient cosines as f32 bits (floor_zero_decode's        *
                                * output); the device computes the curve.  The row's floor needs a    *
                                * floor-0 description (lwb_setup_set_floor0): host floor arrays are   *
                                * refused without one, device ones act as LWB_FLOOR_UNUSED.           */

enum { LWB_OUT_F32_PLANAR = 0,        /* Vec<Vec<f32>>            samples.rs:20-40, 86-90          */
       LWB_OUT_I16_PLANAR = 1,        /* Vec<Vec<i16>>            samples.rs:92-103                */
       LWB_OUT_F32_INTERLEAVED = 2,   /* InterleavedSamples<f32>  samples.rs:43-79                 */
       LWB_OUT_I16_INTERLEAVED = 3,   /* InterleavedSamples<i16>                                   */
       LWB_OUT_F16_PLANAR = 4,        /* Vec<Vec<half::f16>>      a caller's `impl Sample for f16` */
       LWB_OUT_F16_INTERLEAVED = 5,   /* InterleavedSamples<half::f16>                             */
       /* 6 and 7 are not assigned: refused as bad formats */
       LWB_OUT_I32_PLANAR = 8,        /* Vec<Vec<i32>>            a caller's `impl Sample for i32` */
       LWB_OUT_I32_INTERLEAVED = 9,   /* InterleavedSamples<i32>                                   */
       LWB_OUT_I24_PLANAR = 10,       /* Vec<Vec<[u8; 3]>>        packed little-endian 24-bit      */
       LWB_OUT_I24_INTERLEAVED = 11 };/* InterleavedSamples<[u8; 3]>  (S24_3LE)                    */
/* F16 formats: each element is an IEEE binary16 (2 bytes, the layout of the F32 / I16 format of the same arrangement)
 * equal to the binary32 sample x that the F32 format would write, rounded to nearest even: binary16 subnormals are
 * kept (no flush to zero), |x| >= 65520 becomes +-inf, a NaN gives a NaN.  They take the same batch paths as the I16
 * formats of the same layout.  Added under ABI 3 (no struct changes): a library without them refuses out_format 4 / 5
 * with LWB_ERR_INVALID ("bad out_format") before it touches any chain result, stream state or arena -- as every
 * library refuses any out_format above the last one it knows -- so a caller detects support by one refused call. */
/* I32 and I24 formats: samples.rs:92-103 (`Sample for i16`) with the scale changed, as a caller's `impl Sample for i32`
 * writes it with Rust's saturating `as` casts.  I32: y = x * 2147483648.0f (one binary32 multiply, exact), y >= 2^31
 * (x == 1.0 included) gives INT32_MAX, y < -2^31 gives INT32_MIN, NaN gives 0, anything else truncates toward zero; an
 * element is an int32_t.  I24: y = x * 8388608.0f, above 8388607 gives 8388607, below -8388608 gives -8388608, NaN gives
 * 0, anything else truncates toward zero; an element is the low 3 bytes of that integer, little-endian two's
 * complement, with no padding (element offsets and strides count 3-byte samples).  Both take the batch paths of the
 * F32 / I16 formats of the same layout, except that a planar I24 batch takes the fused kernels only when its rows start at
 * element offsets (and strides) that are multiples of 16 -- 48 bytes, a 16-byte boundary.  Added under ABI 3 (no
 * struct changes), refused as the F16 formats are by a library without them; 6 and 7 stay unassigned and refused. */

typedef struct lwb_packet {
    uint8_t mode_number;             /* audio.rs:925                                               */
    uint8_t prev_window_flag;        /* audio.rs:935, long blocks only (ignored for short ones)    */
    uint8_t next_window_flag;
    uint8_t reserved;
    const uint8_t *floor_kind;       /* [channels] LWB_FLOOR_*                                     */
    const uint32_t *floor1_y;        /* [channels][LWB_MAX_POSTS] rows used where kind == ONE      */
    const float *dense_floor;        /* [channels][n/2], rows used where kind == DENSE, else NULL  */
    const float *residue;            /* [channels][n/2] after residue_packet_decode (audio.rs:986) */
} lwb_packet;

/* Synchronous convenience = submit + flush + fetch.  out: planar [channels][capacity] or
 * interleaved [capacity][channels] (channels: lwb_setup_output_channels); *n_samples = samples per channel written (0 for the first
 * packet after a reset).  Host buffers. */
int lwb_decode_packet(lwb_stream *s, const lwb_packet *pkt, int out_format, void *out,
                      size_t capacity_per_channel, size_t *n_samples);
/* Entry at record_pre_mdct (audio.rs:1041): spectrum [channels][n/2] already floor x residue. */
int lwb_decode_spectrum(lwb_stream *s, uint8_t mode_number, int prev_window_flag,
                        int next_window_flag, const float *spectrum, int out_format, void *out,
                        size_t capacity_per_channel, size_t *n_samples);

/* ---- batches: many streams x consecutive packets in one submission ------------------------- */
enum { LWB_ENTRY_SPECTRUM = 0,   /* coeffs = floor x residue, enters at audio.rs:1041             */
       LWB_ENTRY_RESIDUE = 1,    /* coeffs = residue vectors, enters at audio.rs:988               */
       LWB_ENTRY_VQ = 2 };       /* no dense coefficients cross the boundary: the residue vectors are  *
                                  * accumulated on the device from the packets' VQ entry indices       *
                                  * (audio.rs:587-717); coeff_offset still lays out the (device-only)   *
                                  * coefficient arena.  Needs the setup's codebooks / residues, <= 8     *
                                  * channels, channels * n/2 <= 12288, VQ books of <= 65536 entries whose   *
                                  * dimension divides their residue's partition size.  Every batch shape  *
                                  * runs on the kernels of its dense LWB_ENTRY_RESIDUE twin: k_long, the  *
                                  * segmented schedules, k_mid, and k_chain for the rest (interleaved     *
                                  * output, other blocksizes), which accumulates in shared memory itself. */
/* The VQ vectors of a packet's residue, in the order the entropy decoder produces them (SURVEY.md 8f rank 2), as RUNS:
 * one run = the consecutive vectors one residue_packet_read_partition call reads (audio.rs:587-618) -- same codebook,
 * same pass, positions in arithmetic progression -- plus one 16-bit codebook entry per vector in a side array.  The
 * f32 += order of the reference is kept on the device: per coefficient the contributions are added pass by pass
 * (audio.rs:595, :611); within a pass no two vectors of a packet touch the same coefficient. */
typedef struct lwb_vq_run {
    uint16_t pos;                    /* where vector 0 of the run lands (see kind)                          */
    uint16_t first;                  /* index of its entry in the packet's slice of vq_entries              */
    uint8_t book;                    /* codebook index                                                      */
    uint8_t pass_kind;               /* bits 0..2 pass (0..7), bits 3..4 kind:                                *
                                      *   0 contiguous in a channel vector (residue type 1): pos = channel * n/2 + bin,
                                      *     vector i at pos + i * dimensions
                                      *   1 strided (type 0, audio.rs:589-597): vector i at pos + i, its value j at
                                      *     + j * step, step = partition_size(aux) / dimensions
                                      *   2 interleaved (type 2, audio.rs:744-756): pos indexes the interleaved vector of
                                      *     submap `aux` (element t = channel t % ch, bin t / ch), vector i at pos + i * dimensions */
    uint8_t aux;                     /* kind 1: residue index; kind 2: submap index                          */
    uint8_t count;                   /* vectors in the run (a longer partition is split)                     */
} lwb_vq_run;
#define LWB_VQ_PASS_KIND(pass, kind) ((uint8_t)((pass) | ((kind) << 3)))
enum { LWB_MEM_HOST = 0, LWB_MEM_DEVICE = 1 };

/* One stream's run of consecutive packets.  Input arenas are chain-major: the chain's packets
 * follow each other, each packet as [channels][n/2 of that packet].
 * Output: a chain writes exactly n_samples elements per channel plane at out_offset + c * out_stride
 * (planar), or n_samples * channels elements at out_offset (interleaved), and nothing else in `pcm`
 * (channels: lwb_setup_output_channels of the stream's setup),
 * in either memory space: the gaps between planes and between chains keep what the caller put there.
 * Any element offsets and any pointer alignment are accepted, as long as every range a chain touches ends
 * inside the 64-bit address space: a chain whose PCM write set (out_offset + (channels - 1) * out_stride +
 * n_samples, or out_offset + n_samples * channels), coefficient range or packet-row range, counted in bytes,
 * would wrap past 2^64 is refused with LWB_ERR_BUFFER before anything is queued.  The fused kernels take device-memory
 * batches whose coeffs / dense_floor / pcm are 16-byte aligned and whose coeff_offset, out_offset and
 * out_stride are multiples of 4 (host-memory batches: the offsets only); anything else runs on the
 * chain kernel, which gives the same results more slowly. */
typedef struct lwb_chain {
    lwb_stream *stream;
    uint32_t n_packets;
    const uint8_t *mode_numbers;      /* [n_packets] (host memory)                                 */
    const uint8_t *prev_window_flags; /* [n_packets] or NULL = all 1                               */
    const uint8_t *next_window_flags; /* [n_packets] or NULL = all 1                               */
    uint64_t coeff_offset;            /* element offset of the chain's first packet in `coeffs`    */
    uint64_t packet_index;            /* index of the chain's first packet in per-packet arenas    */
    uint64_t out_offset;              /* element offset of the chain's PCM in `pcm`                 */
    uint64_t out_stride;              /* planar: elements between channel planes (>= total samples)*/
    /* results */
    uint32_t n_samples;               /* samples per channel written by this chain (produced, less what the stream's
                                       * window, lwb_stream_set_window, leaves out)                 */
    uint32_t packets_done;            /* == n_packets unless status != 0                           */
    int32_t status;                   /* LWB_OK or the error of packet `packets_done`              */
} lwb_chain;

/* A host-memory batch (memory == LWB_MEM_HOST) is staged on the device as its extent: coefficient elements from the
 * lowest coeff_offset to the highest coefficient end, PCM elements from the lowest out_offset to the highest end of a
 * write set, gaps included.  Its device memory grows with that span, not with the samples decoded: two chains 2^33
 * elements apart, or one planar chain with an out_stride of 2^32, stage 32 GiB of f32 PCM.  Keep the chains of one
 * host-memory batch close together in the arenas. */
typedef struct lwb_batch_io {
    int entry;                        /* LWB_ENTRY_*                                               */
    int memory;                       /* LWB_MEM_*: where coeffs/dense_floor/pcm live              */
    const float *coeffs;              /* spectrum or residue arena                                 */
    const float *dense_floor;         /* same layout as coeffs, or NULL (LWB_ENTRY_RESIDUE)        */
    const uint8_t *floor_kind;        /* [total_packets][channels]   (LWB_ENTRY_RESIDUE), see floor_memory */
    const uint32_t *floor1_y;         /* [total_packets][channels][LWB_MAX_POSTS], see floor_memory */
    int out_format;                   /* LWB_OUT_*                                                 */
    void *pcm;                        /* output arena                                              */
    /* LWB_ENTRY_VQ: the runs / entries of packet row r (= chain.packet_index + k); all four arrays live where the    *
     * floor arrays live (floor_memory).                                                                            */
    const lwb_vq_run *vq_runs;
    const uint64_t *vq_run_offsets;   /* [total_packets + 1]: packet row r owns vq_runs[off[r] .. off[r + 1])          */
    const uint16_t *vq_entries;
    const uint64_t *vq_entry_offsets; /* [total_packets + 1]: ... and vq_entries[eoff[r] .. eoff[r + 1])            */
    int floor_memory;                 /* LWB_MEM_*: where floor_kind / floor1_y live (0 = host).   *
                                       * Device arrays are read in place (nothing is uploaded, and   *
                                       * nothing about them can be validated on the host: a kind    *
                                       * outside LWB_FLOOR_* acts as LWB_FLOOR_UNUSED); a decode     *
                                       * server whose entropy stage fills device-visible buffers     *
                                       * submits residue-entry batches without any per-step copy.   */
} lwb_batch_io;

/* All chains must use setups with the same channel count per chain's own stream; chains may
 * mix setups.  Returns LWB_OK when the batch ran (per-chain status holds format errors), or a
 * CUDA / argument error.  With LWB_MEM_HOST the call returns after the PCM has landed in `pcm`;
 * with LWB_MEM_DEVICE it returns after the launches are enqueued on lwb_ctx_cuda_stream().  Such a batch's host-memory
 * floor / VQ arrays (floor_memory == LWB_MEM_HOST) are uploaded by copies queued on that stream, which read them when
 * the stream reaches them, as cudaMemcpyAsync reads pinned memory: keep them unchanged until the batch's work has run
 * (lwb_ctx_synchronize, or an event recorded on the stream after the call).  The chain array and the mode and flag
 * arrays are read before the call returns.  A batch that is refused changes no chain result and no stream state. */
int lwb_decode_chains(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io);

/* Asynchronous batches.  A decode server that feeds the GPU from host memory queues batch k + 1 (and entropy-decodes
 * on the same thread) while batch k runs: the host-to-device copies of one batch overlap the kernels and copies of the
 * one before it, and nothing drains between calls.
 *
 * lwb_submit_chains queues the batch like lwb_decode_chains and returns without waiting for it; *ticket identifies its
 * work.
 * Before it returns:
 *   - it makes the same argument checks and refusals as lwb_decode_chains, with the same codes and messages;
 *   - the per-chain results (n_samples, packets_done, status) are written;
 *   - the stream states advance, so a stream can appear in the next submit at once, with its packets in order;
 *   - the chain array and the mode and flag arrays have been read.
 * A submit that is refused (an argument or memory check, a batch lwb_decode_chains would refuse) changes no chain
 * result, no stream state and no arena.  After LWB_ERR_CUDA the chain results are not written and no stream state is
 * committed on the host, but kernels already queued may have run: the device-side state of the batch's streams is
 * undefined (reset or re-import them).  The staging a failed batch took is reused only behind what it had queued.
 * Until the ticket completes:
 *   - LWB_MEM_HOST: `pcm` is written only when the ticket completes.  The caller keeps `coeffs`, `dense_floor` and
 *     the host floor / VQ arrays unchanged and does not read `pcm`.
 *   - LWB_MEM_DEVICE: the call is lwb_decode_chains plus a ticket (see there for host floor arrays).
 * Page-locked memory only: every array of a host-memory submit (coeffs, dense_floor, pcm and, with floor_memory ==
 * LWB_MEM_HOST, the floor and VQ arrays) must be page-locked -- from lwb_host_alloc, cudaHostAlloc or cudaHostRegister
 * -- at the first and the last byte the batch touches.  Pageable memory is refused with LWB_ERR_INVALID before any
 * state or result changes (a bounce copy would hide a whole extra pass over the data; lwb_decode_chains takes it).
 * Tickets complete in submission order.  0 is never issued.  Any ticket up to the newest one issued may be queried or
 * waited on, at any age.
 * A submit still blocks the calling thread in these places, and nowhere else:
 *   - arena growth: a staging arena of a host set grows after that set's previous ticket has completed; the
 *     context's other arenas grow after the compute stream has drained;
 *   - staging-ring wrap: descriptors are written to pinned staging that waits for the copy three stagings back.  The
 *     four-kernel path (batches of more than 8 channels or with buffers beyond shared memory) stages once per round of
 *     its IMDCT scratch, so a batch of more than three rounds waits at its fourth round for its own first copy.
 * lwb_ctx_synchronize, lwb_ctx_destroy and lwb_stream_destroy wait for every queued copy as well as every kernel. */
int lwb_submit_chains(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, uint64_t *ticket);
/* *done = 1 once every copy and kernel of `ticket` has finished (a host-memory batch's PCM is in `pcm`), else 0.
 * Never blocks. */
int lwb_ticket_query(lwb_ctx *ctx, uint64_t ticket, int *done);
/* Blocks until `ticket` has finished.  LWB_ERR_CUDA if its work failed asynchronously. */
int lwb_ticket_wait(lwb_ctx *ctx, uint64_t ticket);

/* Prepared batches.  A decode server submits the same batch shape step after step (same streams,
 * same packets per stream, same arenas); planning it again each time costs more host time than
 * the GPU needs to run it.  lwb_plan_create captures the chain array, the io block and the
 * per-chain mode / flag arrays BY REFERENCE (they must stay valid and unchanged until
 * lwb_plan_destroy); lwb_plan_execute is then equivalent to lwb_decode_chains on that batch
 * -- same results, same stream-state updates, same per-chain outputs in the captured chain
 * array -- but reuses the device descriptors whenever no stream state has changed shape since they
 * were built (it re-plans by itself otherwise, e.g. on the first execution after a reset). */
typedef struct lwb_plan lwb_plan;
int lwb_plan_create(lwb_ctx *ctx, lwb_chain *chains, size_t n_chains, const lwb_batch_io *io, lwb_plan **out);
int lwb_plan_execute(lwb_plan *plan);
void lwb_plan_destroy(lwb_plan *plan);

/* Debug taps at the reference's record_* points (lib.rs:56-94; audio.rs:1004, 1041, 1054):
 * run one packet and return the intermediate vectors instead of PCM.  taps: any may be NULL.
 * post_inverse / pre_mdct: [channels][n/2]; post_mdct: [channels][n].  Does not touch the state. */
int lwb_debug_packet_taps(lwb_stream *s, const lwb_packet *pkt, float *post_inverse,
                          float *pre_mdct, float *post_mdct);

#ifdef __cplusplus
}
#endif
#endif /* LEWTON_B200_H */
