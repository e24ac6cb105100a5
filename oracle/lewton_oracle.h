/*
 * lewton_oracle.h -- CPU restatement of lewton's packet-synthesis arithmetic.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library, and only as the checker / the timed CPU baseline.
 * The product (lewton_b200/) never links, imports or calls it.
 *
 * Why a restatement: the reference (RustAudio/lewton @ bb2955b, v0.10.2) is pure
 * Rust and this project is built without a Rust toolchain, so the reference is
 * not compiled (oracle/_ref is therefore absent).  Each function below cites the
 * reference file:line whose arithmetic it follows, operation for operation, in
 * IEEE binary32 without contraction (-ffp-contract=off, no -ffast-math).
 *
 * Pinning: tests/test_oracle_golden.py checks this library against every
 * fixture the reference's own tests hold for the path (the JSON files under tests/golden,
 * extracted by tests/golden/make_golden.py): IMDCT ARR_1 (5e-5, the
 * reference's own tolerance), ARR_2 (5e-5), ARR_3 (5e-4), the blocksize-8
 * bitreverse table, the 17 render_point triples and the 25 neighbour cases.
 * Stages the reference itself never unit-tests (render_line, coupling, window,
 * overlap-add, i16 quantise) are pinned only by fidelity to the cited lines
 * plus independent mathematical checks (f64 DCT-IV, TDAC round trip).
 */
#ifndef LEWTON_ORACLE_H
#define LEWTON_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LWO_MAX_POSTS 65
#define LWO_MAX_CHANNELS 255

/* header_cached.rs:20-41  TwiddleFactors + CachedBlocksizeDerived */
typedef struct lwo_tables {
    int bs;            /* log2 blocksize, 6..13 */
    int n;             /* 1 << bs */
    float *a;          /* [n/2] */
    float *b;          /* [n/2] */
    float *c;          /* [n/4] */
    float *window;     /* [n/2] window_slope */
    uint32_t *bitrev;  /* [n/8] */
} lwo_tables;

lwo_tables *lwo_tables_new(int bs);                 /* header_cached.rs:34-40 */
void lwo_tables_free(lwo_tables *t);
const float *lwo_tables_a(const lwo_tables *t);
const float *lwo_tables_b(const lwo_tables *t);
const float *lwo_tables_c(const lwo_tables *t);
const float *lwo_tables_window(const lwo_tables *t);
const uint32_t *lwo_tables_bitrev(const lwo_tables *t);

/* imdct.rs:291-659; buffer has n floats, the first n/2 hold the spectrum. */
void lwo_inverse_mdct(const lwo_tables *t, float *buffer);
/* audio.rs:792-825 (definition-level cross-check, f32 like the reference) */
void lwo_inverse_mdct_slow(float *buffer, int n);
/* same definition evaluated in double precision (independent check) */
void lwo_inverse_mdct_f64(const float *spectrum, double *out, int n);

/* audio.rs:253-292; return 0 on success, -1 where the reference panics */
int lwo_low_neighbor(const uint32_t *v, int x, int *idx, uint32_t *val);
int lwo_high_neighbor(const uint32_t *v, int x, int *idx, uint32_t *val);
/* audio.rs:354-367 */
uint32_t lwo_render_point(uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1, uint32_t x);

/* header.rs:415-424 (the fields the synthesis half uses) */
typedef struct lwo_floor1 {
    int multiplier;                       /* 1..4 */
    int nposts;                           /* floor1_x_list.len(), 2..65 */
    uint32_t x_list[LWO_MAX_POSTS];       /* floor1_x_list */
    int sorted_idx[LWO_MAX_POSTS];        /* floor1_x_list_sorted[i].0 */
} lwo_floor1;

/* header.rs:887-889: fill sorted_idx from x_list (stable sort by x) */
void lwo_floor1_sort(lwo_floor1 *fl);
/* audio.rs:391-435; returns 0, or -1 where the reference would panic */
int lwo_floor1_amplitude(const lwo_floor1 *fl, const uint32_t *floor1_y,
                         uint32_t *final_y, uint8_t *step2);
/* audio.rs:503-555; writes n2 floats; returns 0 */
int lwo_floor1_synthesis(const lwo_floor1 *fl, const uint32_t *final_y,
                         const uint8_t *step2, int n2, float *out);
/* integer curve before the dB table (for bisecting) */
int lwo_floor1_curve_y(const lwo_floor1 *fl, const uint32_t *final_y,
                       const uint8_t *step2, int n2, uint32_t *out_y);
const float *lwo_inverse_db_table(void);  /* audio.rs:437-501 */

/* audio.rs:762-777 applied over len bins */
void lwo_inverse_couple(float *mag, float *ang, int len);

/* samples.rs:92-103 */
int16_t lwo_sample_i16(float v);

/* audio.rs:1056-1073 / 889-908 */
typedef struct lwo_window_geom {
    int n, left_start, left_end, right_start, right_end, left_use_bs1;
} lwo_window_geom;
void lwo_window_geometry(int bs0, int bs1, int blockflag, int prev_flag, int next_flag,
                         lwo_window_geom *g);

/* audio.rs:847-861 PreviousWindowRight */
typedef struct lwo_pwr {
    int has;            /* data.is_some() */
    int channels;
    int len;            /* per-channel length (all equal) */
    float *data;        /* [channels][cap] */
    int cap;
} lwo_pwr;
lwo_pwr *lwo_pwr_new(int channels, int cap);
void lwo_pwr_reset(lwo_pwr *p);
void lwo_pwr_free(lwo_pwr *p);
int lwo_pwr_has(const lwo_pwr *p);
int lwo_pwr_len(const lwo_pwr *p);
float *lwo_pwr_data(lwo_pwr *p, int ch);
void lwo_pwr_set(lwo_pwr *p, int len);   /* mark Some(..) with given per-channel len */

enum { LWO_FLOOR_UNUSED = 0, LWO_FLOOR_ONE = 1, LWO_FLOOR_DENSE = 2 };

/* One packet's post-entropy-decode payload, per channel. */
typedef struct lwo_channel_in {
    int floor_kind;                 /* LWO_FLOOR_* */
    const lwo_floor1 *fl;           /* for LWO_FLOOR_ONE */
    const uint32_t *floor1_y;       /* raw decoded Y values, nposts entries */
    const float *dense_floor;       /* for LWO_FLOOR_DENSE: n/2 floats (floor-0 curve from host) */
    float *residue;                 /* n/2 floats, modified in place by coupling */
} lwo_channel_in;

/* audio.rs:988-1157: the whole back half of read_audio_packet_generic.
 * out[ch] must hold n floats; *out_len receives right_start-left_start or 0.
 * Returns 0 ok, 1 AudioBadFormat (OLA guard audio.rs:1107-1111),
 * 3 channel-count mismatch (a panic in the reference, audio.rs:1086). */
int lwo_synth_packet(const lwo_tables *t0, const lwo_tables *t1, int channels,
                     int blockflag, int prev_flag, int next_flag,
                     int n_coupling, const uint8_t *mag, const uint8_t *ang,
                     lwo_channel_in *chans, lwo_pwr *pwr,
                     float *out /* [channels][n] */, int *out_len);

/* Entry at audio.rs:1041 (record_pre_mdct): spectrum[ch][n/2] already formed. */
int lwo_synth_spectrum(const lwo_tables *t0, const lwo_tables *t1, int channels,
                       int blockflag, int prev_flag, int next_flag,
                       const float *spectrum /* [channels][n/2] */, lwo_pwr *pwr,
                       float *out /* [channels][n] */, int *out_len);

/* CPU baseline (bench.py cpu_baseline / --impl reference): S chains x P
 * long/long blocks, IMDCT + window + OLA, `threads` pthreads, static partition
 * over chains, the pass repeated `reps` times over the same input.  spectrum [S][P][n2];
 * out [S][P*n2].  Returns seconds of the timed region (CLOCK_MONOTONIC), scratch
 * preallocated outside it. */
double lwo_bench_chains(int bs, int chains, int packets, const float *spectrum,
                        float *out, int threads, int reps);

#ifdef __cplusplus
}
#endif
#endif
