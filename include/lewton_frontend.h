/*
 * lewton_frontend.h -- C ABI of the HOST front half that feeds lewton_b200.h: Vorbis header
 * parsing, audio-packet entropy decode up to the cut at audio.rs:986, Ogg paging, and the
 * OggStreamReader-style loop around them (SURVEY.md section 8(f) rank 1 and 3).
 *
 * This is CPU code by nature (bit-serial Huffman / VQ decode); it is the part of lewton that stays
 * on the host in the drop-in design (INTEGRATION.md).  In a Rust build the crate's own front half
 * plays this role; this C++ restatement exists because the project is built without a Rust toolchain,
 * so that whole streams can be decoded end to end and the batch / residue entry points of the
 * CUDA back end can be driven by real bitstreams.
 *
 * Reference interfaces mirrored (file:line in the reference's src/):
 *   lwf_headers_parse            header.rs:221 read_header_ident, :309 read_header_comment,
 *                                :1082 read_header_setup
 *   lwf_packet_decode            audio.rs:919-986 (front half of read_audio_packet_generic),
 *                                :109-158 floor_zero_decode, :160-212 floor_zero_compute_curve,
 *                                :215-251 floor_one_decode, :557-760 floor/residue decode
 *   lwf_decoded_sample_count     audio.rs:874-909 get_decoded_sample_count
 *   lwf_ogg_*                    ogg 0.8.0 PacketReader as used by inside_ogg.rs:16-143
 *   lwf_reader_*                 inside_ogg.rs:60-313 OggStreamReader (read_dec_packet[_itl], skip_samples_linear, seek_absgp_pg,
 *                                end-of-stream truncation :219-222, absgp accounting :223-227,
 *                                chained streams :118-141)
 * Status codes are lewton_b200.h's LWB_* plus the LWF_* header errors below.
 */
#ifndef LEWTON_FRONTEND_H
#define LEWTON_FRONTEND_H

#include <stddef.h>
#include <stdint.h>

#include "lewton_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* header.rs:35-44 HeaderReadError, audio.rs:26-41 AudioReadError (values continue LWB_*) */
enum {
    LWF_ERR_END_OF_PACKET = 16,     /* HeaderReadError::EndOfPacket / AudioReadError::EndOfPacket   */
    LWF_ERR_NOT_VORBIS_HEADER = 17,
    LWF_ERR_UNSUPPORTED_VERSION = 18,
    LWF_ERR_HEADER_BAD_FORMAT = 19,
    LWF_ERR_HEADER_BAD_TYPE = 20,
    LWF_ERR_HEADER_IS_AUDIO = 21,
    LWF_ERR_UTF8 = 22,
    LWF_ERR_AUDIO_IS_HEADER = 23,   /* AudioReadError::AudioIsHeader                               */
    LWF_ERR_OGG = 24,               /* framing: capture pattern, CRC, lacing, truncated page       */
    LWF_ERR_NO_MORE_PACKETS = 25    /* read_packet() == None                                       */
};

/* ---- headers --------------------------------------------------------------------------------- */
typedef struct lwf_headers lwf_headers;     /* IdentHeader + CommentHeader + SetupHeader           */

typedef struct lwf_info {                   /* header.rs:188-211 IdentHeader + setup counts        */
    uint8_t audio_channels, blocksize_0, blocksize_1;
    uint32_t audio_sample_rate;
    int32_t bitrate_maximum, bitrate_nominal, bitrate_minimum;
    uint32_t n_codebooks, n_floors, n_residues, n_mappings, n_modes, n_comments;
} lwf_info;

int lwf_headers_parse(const uint8_t *ident, size_t ident_len, const uint8_t *comment, size_t comment_len,
                      const uint8_t *setup, size_t setup_len, lwf_headers **out);
void lwf_headers_destroy(lwf_headers *h);
int lwf_headers_info(const lwf_headers *h, lwf_info *out);
/* vendor string (index < 0) or "key=value" of comment `index`; returns the length, copies <= cap */
size_t lwf_headers_comment(const lwf_headers *h, int index, char *buf, size_t cap);
/* what lwb_setup_create needs, filled from the parsed headers (tables via lwb_tables_generate) */
int lwf_headers_make_setup(const lwf_headers *h, lwb_ctx *ctx, lwb_setup **out);
/* the same, and every type-0 floor that can travel as an LWB_FLOOR_ZERO record (order 2..63, nonzero rate and bark
 * map size) described with lwb_setup_set_floor0: the setup for packets decoded with LWF_DECODE_FLOOR0_RECORDS */
int lwf_headers_make_setup_floor0(const lwf_headers *h, lwb_ctx *ctx, lwb_setup **out);

/* ---- one audio packet: front half of read_audio_packet_generic ------------------------------- */
typedef struct lwf_decoded_packet {
    uint8_t mode_number;
    uint8_t blockflag;
    uint8_t prev_window_flag, next_window_flag;    /* 1 for short blocks (map_or(true, ..))        */
    uint32_t n;                                     /* blocksize of this packet                     */
    /* per channel, caller-provided storage: */
    uint8_t *floor_kind;        /* [channels]                LWB_FLOOR_*                            */
    uint32_t *floor1_y;         /* [channels][LWB_MAX_POSTS]                                        */
    float *dense_floor;         /* [channels][n/2]: floor-0 curves (only rows with LWB_FLOOR_DENSE) */
    float *residue;             /* [channels][n/2]: residue vectors before inverse coupling         */
} lwf_decoded_packet;

/* Buffers in `out` must hold channels x blocksize_1/2 floats.  Returns LWB_OK, LWF_ERR_AUDIO_IS_HEADER,
 * LWF_ERR_END_OF_PACKET (header bits missing) or LWB_ERR_BAD_FORMAT (audio.rs:926-930, :975). */
int lwf_packet_decode(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out);
/* flags: LWF_DECODE_FLOOR0_RECORDS -- type-0 floors of order <= 63 (and nonzero rate / bark map size) come out as
 * LWB_FLOOR_ZERO records in their floor1_y row instead of dense curves, for a setup from lwf_headers_make_setup_floor0;
 * dense_floor may then be NULL when no type-0 floor of the stream needs it.  flags == 0 is lwf_packet_decode. */
enum { LWF_DECODE_FLOOR0_RECORDS = 1 };
int lwf_packet_decode_ex(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out, int flags);
int lwf_decoded_sample_count(const lwf_headers *h, const uint8_t *packet, size_t len, size_t *n_samples);
/* The same front half with the residue left as VQ runs + entries (SURVEY.md 8f rank 2; audio.rs:587-717): what
 * residue_packet_decode would have ADDED, partition by partition in decode order, for LWB_ENTRY_VQ batches (out->residue
 * is not touched and may be NULL).  LWB_ERR_BUFFER if the capacities do not suffice (a packet of L bytes never needs
 * more than 8 L of either).  lwf_headers_vq_capable: 1 if the stream qualifies (<= 8 channels, channels * n/2 <= 12288,
 * VQ books of <= 65536 entries whose dimension divides their residue's partition size), else the dense path is used. */
int lwf_headers_vq_capable(const lwf_headers *h);
int lwf_packet_decode_vq(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out,
                         lwb_vq_run *runs, size_t run_capacity, size_t *n_runs, uint16_t *entries, size_t entry_capacity,
                         size_t *n_entries);
int lwf_packet_decode_vq_ex(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out,
                            lwb_vq_run *runs, size_t run_capacity, size_t *n_runs, uint16_t *entries, size_t entry_capacity,
                            size_t *n_entries, int flags);

/* ---- Ogg paging -------------------------------------------------------------------------------- */
typedef struct lwf_ogg lwf_ogg;             /* PacketReader over a memory buffer (not copied)      */
typedef struct lwf_ogg_packet {
    const uint8_t *data;                    /* valid until the next lwf_ogg_next_packet             */
    size_t len;
    uint32_t stream_serial;
    uint64_t absgp_page;
    uint8_t first_in_stream, last_in_stream, first_in_page, last_in_page;
} lwf_ogg_packet;
int lwf_ogg_open(const uint8_t *data, size_t len, lwf_ogg **out);
void lwf_ogg_close(lwf_ogg *o);
int lwf_ogg_next_packet(lwf_ogg *o, lwf_ogg_packet *pkt);    /* LWF_ERR_NO_MORE_PACKETS at the end  */

/* ---- OggStreamReader --------------------------------------------------------------------------- */
typedef struct lwf_reader lwf_reader;
/* Reads the three headers, builds the device-side setup on `ctx`, opens a PreviousWindowRight. */
int lwf_reader_open(lwb_ctx *ctx, const uint8_t *data, size_t len, lwf_reader **out);
void lwf_reader_close(lwf_reader *r);
const lwf_headers *lwf_reader_headers(const lwf_reader *r);
/* read_dec_packet_generic: decodes the next audio packet through lwb_decode_packet.  `out_format`
 * LWB_OUT_*; `out` holds capacity_total elements in all: planar channel c starts at
 * c * (capacity_total / channels), with the channel count of the stream the packet belongs to (a
 * chained stream may change it: query lwf_reader_headers afterwards).  *n_samples = samples per
 * channel after end-of-stream truncation.  LWF_ERR_NO_MORE_PACKETS = Ok(None). */
int lwf_reader_read_dec_packet(lwf_reader *r, int out_format, void *out, size_t capacity_total,
                               size_t *n_samples);
int lwf_reader_last_absgp(const lwf_reader *r, uint64_t *absgp);   /* returns 0 and sets *absgp if Some */
/* skip_samples_linear (inside_ogg.rs:244-283): walks packets by their sample counts only, decodes the packet before
 * the target on a fresh PreviousWindowRight (dropped) and returns the target packet.  *got_packet = 0 <=> Ok((None, _))
 * (the stream ended first); *left_to_skip = the second element of the reference's tuple. */
int lwf_reader_skip_samples_linear(lwf_reader *r, size_t to_skip, int out_format, void *out, size_t capacity_total,
                                   size_t *n_samples, size_t *left_to_skip, int *got_packet);
/* seek_absgp_pg (inside_ogg.rs:307-313): page-granular seek inside the current logical stream to a position <= absgp;
 * afterwards get_last_absgp() is None and the next packet returns 0 samples (fresh PreviousWindowRight). */
int lwf_reader_seek_absgp_pg(lwf_reader *r, uint64_t absgp);

/* ---- many streams at once: host entropy decode on a thread pool, one batched synthesis call ---- */
/* The shape of a decode server (BASELINE configs 1/3 at scale): packets of many logical streams that
 * share one set of headers are entropy-decoded in parallel on the host straight into pinned arenas
 * (residue vectors, floor posts), then synthesised by ONE lwb_decode_chains call (residue entry,
 * host memory).  Streams are independent; packets within a stream keep their order. */
typedef struct lwf_stream_job {
    lwb_stream *stream;               /* PreviousWindowRight of this logical stream                  */
    uint32_t n_packets;
    const uint8_t *const *packets;    /* [n_packets] audio packets in stream order                   */
    const size_t *lengths;            /* [n_packets]                                                 */
    uint64_t out_offset;              /* element offset of this stream's PCM in `pcm`                */
    uint64_t out_stride;              /* planar formats: elements between channel planes             */
    /* results */
    uint32_t n_samples;               /* samples per channel written (less what the stream window, lwb_stream_set_window, drops) */
    uint32_t packets_done;            /* packets synthesised (== n_packets unless status != 0)       */
    int32_t status;                   /* LWB_OK, or the error of packet `packets_done`               */
} lwf_stream_job;

typedef struct lwf_batcher lwf_batcher;
/* `setup` must come from lwf_headers_make_setup(h, ctx); threads <= 0: one per host CPU */
int lwf_batcher_create(lwb_ctx *ctx, const lwf_headers *h, int threads, lwf_batcher **out);
/* waits for the submitted batches that still read the batcher's arenas, then frees them */
void lwf_batcher_destroy(lwf_batcher *b);
/* Jobs whose stream was opened on `setup` are entropy-decoded with `h` (which, like the batcher's own headers, must
 * outlive the batcher).  Streams of any setup not registered here keep the headers given to lwf_batcher_create, as
 * before.  LWB_ERR_INVALID: NULL argument, a setup already registered, a setup whose channel count or blocksizes differ
 * from h's ident header (or that was made on another context), or (LWB_ENTRY_VQ) headers that fail
 * lwf_headers_vq_capable.
 * Header sets are grouped by (channel count, blocksize_0, blocksize_1); the batcher's own headers form a group too.  A
 * decode or submit entropy-decodes all its jobs in one parallel pass, then synthesises each group's jobs as one batch
 * (a residue or VQ batch has one channel count, and a batch of one blocksize pair runs whole on that shape's fused
 * kernel).  With no header set added there is one group, and every call makes the batches it made before. */
int lwf_batcher_add_headers(lwf_batcher *b, const lwf_headers *h, const lwb_setup *setup);
/* LWB_ENTRY_RESIDUE (default: dense residue vectors cross the boundary) or LWB_ENTRY_VQ (VQ records do; needs
 * lwf_headers_vq_capable of the batcher's headers and of every header set added) */
int lwf_batcher_set_entry(lwf_batcher *b, int entry);
/* records != 0: decode with LWF_DECODE_FLOOR0_RECORDS (the jobs' streams must come from lwf_headers_make_setup_floor0);
 * applies to every header set.  A group whose type-0 floors all qualify allocates and sends no dense floor arena. */
int lwf_batcher_set_floor0(lwf_batcher *b, int records);
/* Returns once the PCM has landed in `pcm` (host memory, pageable or page-locked).  It first waits for every batch
 * lwf_batcher_submit queued that still reads the batcher's arenas. */
int lwf_batcher_decode(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm);
/* Asynchronous lwf_batcher_decode.  Entropy-decodes `jobs` like lwf_batcher_decode, queues their synthesis as ONE
 * lwb_submit_chains batch per group of header sets (lwf_batcher_add_headers), back to back, on the batcher's ctx and
 * returns once they are queued.  pcm_memory: LWB_MEM_HOST (`pcm` must be page-locked, as for a host-memory
 * lwb_submit_chains) or LWB_MEM_DEVICE (`pcm` is device memory of the batcher's ctx; the PCM never crosses to the
 * host).  *ticket is a ticket of that ctx, the last group's (tickets complete in submission order, so it covers every
 * batch of the call): wait or query it with lwb_ticket_wait / lwb_ticket_query; `pcm` holds the PCM once it has
 * completed.
 * Before it returns:
 *   - the entropy decode is finished: the jobs' packet buffers may be reused or freed;
 *   - every job's n_samples, packets_done and status is written, with the values lwf_batcher_decode would give, entropy
 *     and packet-header errors included;
 *   - the stream states have advanced, so a stream can appear in the next submit at once.
 * A refused submit (a NULL argument, a pcm_memory other than the two values, an unknown out_format, pageable host PCM,
 * anything lwb_submit_chains refuses) changes no job result and no stream state, writes nothing to `pcm` and issues no
 * ticket.  With several groups, every group's batch is checked (page-locked PCM included) and every arena grown before
 * the first is queued.  Only LWB_ERR_CUDA or LWB_ERR_BUFFER can then stop a later group's batch: the call returns it
 * without a ticket; the groups queued before it have written their jobs' results and advanced their streams
 * (lwb_ctx_synchronize waits for their PCM), the device-side states of the failing group's streams are undefined, and
 * the jobs and streams of the groups after it are unchanged.
 * Device PCM: the batch reads the residue vectors (LWB_ENTRY_RESIDUE) and dense floor-0 curves from device arenas of
 * the batcher, into which the call copies its pinned ones on lwb_ctx_cuda_stream(); floor and VQ arrays are uploaded by
 * the library as for any device batch with host floor arrays.  The fused kernels take it under the same alignment rule
 * as any device batch (lwb_chain); anything else runs on the chain kernel.
 * Arena sets: the batcher's pinned input arenas, and their device copies, form a ring of two sets (each with one arena
 * per group).  A submit writes the set the submit two back read, after that submit's ticket has completed.
 * A submit blocks the calling thread in these places, and in those lwb_submit_chains lists:
 *   - the entropy decode of the jobs, on the batcher's thread pool;
 *   - arena-set wait: with two submits in flight, a third waits for the ticket of the older one;
 *   - arena growth: a device arena grows after the ctx's stream has drained. */
int lwf_batcher_submit(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory,
                       uint64_t *ticket);
/* wall-clock seconds of the last lwf_batcher_decode: host entropy decode, synthesis call; of the last
 * lwf_batcher_submit: entropy decode, the rest of the call (arena-set wait, uploads and lwb_submit_chains) */
void lwf_batcher_last_timing(const lwf_batcher *b, double *entropy_seconds, double *synthesis_seconds);
/* bytes of the host arrays the last lwf_batcher_decode or lwf_batcher_submit handed to the synthesis (residues or VQ
 * records, dense floor-0 curves, floor kinds and floor1_y rows): what its batches copy to the device */
uint64_t lwf_batcher_last_input_bytes(const lwf_batcher *b);

/* ---- many OggStreamReaders at once: the reader's semantics on the batcher's synthesis ---------- */
/* Each reader is an lwf_reader over its own bytes; one lwf_readers_read advances many of them.  Their Ogg de-paging and
 * sample counting, then their entropy decode, run on the host thread pool; their synthesis is one lwb_submit_chains
 * batch per group of equal channel count and blocksize pair, as lwf_batcher_submit makes it (residue entry, dense
 * floor-0 curves, as lwf_reader decodes).  Each reader returns exactly what a single lwf_reader would return for the
 * same bytes, for reads (lwf_readers_read), page-granular seeks (lwf_readers_seek_absgp_pg) and linear skips
 * (lwf_readers_skip_samples_linear) in any order. */
typedef struct lwf_readers lwf_readers;     /* many OggStreamReaders on one ctx, one host thread pool */
int lwf_readers_create(lwb_ctx *ctx, int threads, lwf_readers **out);       /* threads <= 0: one per host CPU */
void lwf_readers_destroy(lwf_readers *rs);                                   /* waits for its queued reads */
/* lwf_reader_open for one more reader: reads its headers; `data` is not copied and must outlive the reader.  Readers whose
 * ident and setup header bytes are equal share one parsed setup header (parsed once), one lwb_setup and one header set of
 * the entropy decode; each reader's own lwf_headers holds its comments and gives the shared set's info and decode.  The
 * device setup and the reader's stream state are made by the first lwf_readers_read that reads it. */
int lwf_readers_add(lwf_readers *rs, const uint8_t *data, size_t len, uint32_t *index);
const lwf_headers *lwf_readers_headers(const lwf_readers *rs, uint32_t index); /* the stream its NEXT packet belongs to */
int lwf_readers_last_absgp(const lwf_readers *rs, uint32_t index, uint64_t *absgp); /* as lwf_reader_last_absgp */
/* distinct (ident, setup) header byte pairs among the streams the readers have opened: one lwb_setup each */
uint32_t lwf_readers_setup_count(const lwf_readers *rs);
/* wall-clock seconds of the last accepted lwf_readers_read or lwf_readers_skip_samples_linear: the de-paging and sample
 * counting pass (all rounds of a skip's walk), and the internal batcher's entropy decode and rest of its submit
 * (lwf_batcher_last_timing) */
void lwf_readers_last_timing(const lwf_readers *rs, double *paging_seconds, double *entropy_seconds, double *synthesis_seconds);

typedef struct lwf_read_job {
    uint32_t reader;          /* index from lwf_readers_add; a reader may appear in at most one job per call */
    uint32_t max_packets;     /* read at most this many audio packets (calls of lwf_reader_read_dec_packet)  */
    uint64_t out_offset;      /* element offset of this job's PCM in `pcm`                                  */
    uint64_t out_stride;      /* planar: elements between channel planes                                    */
    uint32_t *packet_samples; /* optional [max_packets]: samples each returned packet wrote (NULL: not wanted) */
    /* results */
    uint32_t n_packets;       /* packets returned (what that many single-reader calls would have returned)   */
    uint32_t n_samples;       /* samples per channel written: the concatenation of those packets' PCM       */
    uint8_t  channels;        /* channel count of the stream the packets belong to                           */
    uint8_t  next_chained;    /* 1: the reader now stands at a new logical stream (headers already read)     */
    uint8_t  ended;           /* 1: no packet left (the single reader's LWF_ERR_NO_MORE_PACKETS)             */
    uint8_t  reserved;
    int32_t  status;          /* LWB_OK, or the code the single reader's call for packet n_packets returned  */
} lwf_read_job;
/* Reads up to max_packets audio packets from each job's reader and queues their synthesis, asynchronously, in the manner
 * of lwf_batcher_submit.
 * Equivalence: the PCM a job writes, and packet_samples, are those of n_packets consecutive lwf_reader_read_dec_packet
 * calls on a single reader over the same bytes, concatenated: written sample j of the job goes to out_offset + c *
 * out_stride + j (planar) or out_offset + j * channels + c (interleaved).  f32 is bit for bit the single reader's (up to
 * the sign of zero and NaN payloads), i16 and f16 exactly.  status, lwf_readers_last_absgp and the absgp accounting, and
 * (but for a chained stream, below) lwf_readers_headers are that reader's after those calls.  Nothing outside the
 * job's n_samples samples per channel is written.
 * Errors: a job stops at its first failing packet.  That packet is consumed, as in the single reader; its code
 * (LWB_ERR_BAD_FORMAT, LWF_ERR_END_OF_PACKET, LWF_ERR_AUDIO_IS_HEADER, an Ogg or header error) goes to status, and the
 * reader's next call continues after it.  A job that reads past the last packet sets ended and keeps status LWB_OK.
 * LWB_ERR_MISMATCH in status: the samples the batch wrote differ from the sum of packet_samples, which come from the
 * packets' headers (window flags that disagree with the block before, and that the synthesis did not refuse); the
 * reader has advanced as the other results say.
 * Chained streams: a job never spans two logical streams, so its layout has one channel count (`channels`).  When the
 * next packet begins a new stream the job stops there and reads the new headers (a header error goes to status), and
 * next_chained is set: lwf_readers_headers then gives the new stream, whose channel count and blocksizes lay out the next
 * job.  That next job decodes and drops the new stream's first audio packet first, as read_next_audio_packet does.
 * End of stream: the last packet is truncated to its page's granule position by the stream's output window
 * (lwb_stream_set_window) set for that job alone: the batch keeps its fused kernel and there is no host pass over PCM.
 * Before it returns, the de-paging and entropy decode are done, every job's results are written and the readers have
 * advanced, so they can be read again at once; *ticket (as lwf_batcher_submit's) completes once the PCM is in `pcm`.
 * pcm_memory, page-locked host memory, tickets, the ring of two arena sets and the places the call blocks are
 * lwf_batcher_submit's.
 * Refusals -- LWB_ERR_INVALID for a NULL rs, jobs, pcm or ticket, n_jobs == 0, a pcm_memory other than LWB_MEM_HOST and
 * LWB_MEM_DEVICE, an unknown out_format, an unknown reader index, a reader in two jobs, a planar job whose out_stride is
 * below max_packets * blocksize_1 / 2 + (blocksize_1 - blocksize_0) / 4 of its reader's stream (the most max_packets
 * packets can return: a long block before a short one returns (3 blocksize_1 - blocksize_0) / 4), and anything
 * lwf_batcher_submit refuses (pageable host PCM among them); or the error of making a reader's device setup or stream -- change no job, reader or PCM element and issue
 * no ticket.  After LWB_ERR_CUDA or LWB_ERR_BUFFER from a later group's batch, the jobs of the groups queued before it
 * have their results and their readers have advanced; the others are unchanged. */
int lwf_readers_read(lwf_readers *rs, lwf_read_job *jobs, size_t n_jobs, int out_format, void *pcm, int pcm_memory,
                     uint64_t *ticket);

/* lwf_reader_seek_absgp_pg for each listed reader: a page-granular seek inside the logical stream the single reader
 * stands in, to the last page whose granule position is <= absgps[k]; afterwards lwf_readers_last_absgp is None and the
 * next packet returns 0 samples.  status[k] gets the single reader's code (LWF_ERR_OGG for a bad page on the way or no
 * page of the stream; the reader's position is then unchanged).  A reader whose last read job ended with next_chained
 * seeks where the single reader would: in the stream before, whose headers lwf_readers_headers gives again.
 * The pages are walked on the host thread pool, one task per reader.  Only host state changes: no GPU work is queued, no
 * ticket is issued, and reads still queued are not waited for (they keep the PCM and states they were queued with).
 * Refusals -- LWB_ERR_INVALID for a NULL rs, readers, absgps or status, n == 0, an unknown reader index or a reader
 * listed twice -- change no reader and no status element. */
int (lwf_readers_seek_absgp_pg)(lwf_readers *rs, const uint32_t *readers, const uint64_t *absgps, size_t n, int32_t *status);

typedef struct lwf_skip_job {
    uint32_t reader;          /* index from lwf_readers_add; a reader may appear in at most one job per call           */
    uint32_t out_channels;    /* channels of room at out_offset (0: the reader's current stream's channel count)      */
    uint64_t to_skip;         /* samples per channel to skip                                                           */
    uint64_t out_offset;      /* element offset of this job's PCM in `pcm`                                             */
    uint64_t out_stride;      /* planar: elements between channel planes; interleaved: room per channel               */
    /* results */
    uint64_t left_to_skip;    /* the second element of skip_samples_linear's tuple                                     */
    uint32_t n_samples;       /* samples per channel of the returned packet                                            */
    uint8_t  got_packet;      /* 1: a packet was returned (Ok((Some, _))); 0: the stream ended first, or status != 0   */
    uint8_t  channels;        /* channel count of the stream the reader stands in afterwards                           */
    uint8_t  reserved[2];
    int32_t  status;          /* LWB_OK or the code the single reader's call returned                                  */
} lwf_skip_job;
/* lwf_reader_skip_samples_linear for each job's reader, with the target packets' synthesis queued asynchronously in the
 * manner of lwf_readers_read.
 * Equivalence: each job returns what one lwf_reader_skip_samples_linear call returns on the same bytes: the target
 * packet's PCM (written sample j goes to out_offset + c * out_stride + j planar, out_offset + j * channels + c
 * interleaved; f32 bit for bit, i16 and f16 exactly), n_samples, left_to_skip (to_skip itself when status != 0), the end
 * of the stream (got_packet = 0, status LWB_OK), errors, and lwf_readers_last_absgp, lwf_readers_headers and the overlap
 * state afterwards.  Nothing outside the job's n_samples samples per channel is written.
 * Passes: the walk that only counts samples runs on the host thread pool.  It stops at a chained stream, whose headers
 * are read between rounds of the pool (they change the readers' shared header sets); it then continues in the new
 * stream after decoding and dropping its first audio packet, as the single reader does.  The synthesis is one batch per
 * group, through the internal batcher, as a read's: a job's chain is the packet before the target and the target on a
 * reset stream state (the packet before returns nothing), or, where the single reader has no packet before it (the
 * first packet of the walk, or a stream's last packet with a known granule position), the target alone on the state the
 * reader stands in -- behind a chained stream's dropped packet if the walk entered one.  A target that is its stream's
 * truncated last packet is cut by the stream's output window, as reads cut it.  A job whose walk ends without a target
 * but after dropping a chained stream's first packet synthesises that packet alone, writing nothing.
 * A job that crossed into a chained stream lays its target out with that stream's channel count and blocksizes; it
 * needs out_channels >= that count, and out_stride >= blocksize_1 / 2 + (blocksize_1 - blocksize_0) / 4 of that stream
 * (planar) or (interleaved) out_channels * out_stride >= its channels times that: otherwise the whole call is refused.
 * pcm_memory, page-locked host memory, tickets, the ring of two arena sets and the places the call blocks are
 * lwf_readers_read's.
 * Refusals -- lwf_readers_read's, with max_packets = 1 for the planar stride rule, out_channels (if not 0) below the
 * reader's channel count, and the crossing rule above -- change no job, reader, stream state or PCM element and issue no
 * ticket (a chained stream's headers read by the refused walk may stay parsed for a later call). */
int (lwf_readers_skip_samples_linear)(lwf_readers *rs, lwf_skip_job *jobs, size_t n_jobs, int out_format, void *pcm,
                                      int pcm_memory, uint64_t *ticket);

/* ---- debug taps (known-answer tests of the reference's unit-test vectors) ---------------------- */
float lwf_debug_float32_unpack(uint32_t v);                          /* bitpacking.rs:304-314        */
uint32_t lwf_debug_lookup1_values(uint32_t entries, uint16_t dims);  /* header.rs:616-649            */
uint8_t lwf_debug_ilog(uint64_t v);                                  /* lib.rs:166-172               */
size_t lwf_debug_read_bits(const uint8_t *data, size_t len, const uint8_t *widths, size_t n, uint64_t *out);
int lwf_debug_huffman(const uint8_t *lengths, size_t n, const uint8_t *data, size_t len, uint32_t *out,
                      size_t max_out, size_t *n_out);                /* huffman_tree.rs:113-214      */
/* timing aid: the n packets decoded `reps` times inside one call (vq != 0: records instead of dense residues);
 * seconds, < 0 on error (profiles/frontend_bench.py) */
double lwf_debug_decode_loop(const lwf_headers *h, const uint8_t *const *packets, const size_t *lens, size_t n, int reps, int vq);

#ifdef __cplusplus
}
#endif
#endif
