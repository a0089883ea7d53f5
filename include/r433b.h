/* r433b.h -- C ABI of the H100 IQ -> pulse-train -> bitbuffer hot path.
 *
 * This is the seam a maintainer of merbanan/rtl_433 binds instead of the per-block calls that
 * push_sdr_flow() makes today (src/r_flow.c:151-161, :198, :206-208, :243, :259, :302):
 *
 *   envelope_detect / magnitude_est_cu8 / magnitude_est_cs16   src/baseband.c:36,65,96
 *   baseband_low_pass_filter                                   src/baseband.c:145
 *   baseband_demod_FM / baseband_demod_FM_cs16                 src/baseband.c:210,303
 *   pulse_detect_package (+ pulse_detect_fsk_*)                src/pulse_detect.c:199
 *   pulse_slicer_{pcm,ppm,pwm,manchester_zerobit,dmc,piwm_raw,piwm_dc,nrzs,osv1,rzi}
 *                                                              src/pulse_slicer.c:68-918
 *   run_ook_demods / run_fsk_demods / account_event            src/r_api.c:438-550, src/pulse_slicer.c:26
 *
 * Plain C, plain pointers and sizes; no CUDA or torch types.  One context per GPU, not
 * thread-safe (the reference's decoders are not re-entrant either).  Every function returns
 * 0 on success or a negative R433B_E* code; r433b_last_error() explains the last failure.
 * There is NO CPU fallback: without a usable CUDA device r433b_create() fails.
 */
#ifndef R433B_H_
#define R433B_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define R433B_OK 0
#define R433B_EINVAL (-1)   /* bad argument */
#define R433B_ECUDA (-2)    /* CUDA runtime error, see r433b_last_error() */
#define R433B_ENOMEM (-3)   /* host or device allocation failed */
#define R433B_EOVERFLOW (-4) /* a result arena was too small even after regrowth */
#define R433B_ESTATE (-5)   /* call sequence error (e.g. fetch before process) */

#define R433B_FMT_CU8 2  /* bytes per IQ sample; dm_state.sample_size, include/r_private.h:39 */
#define R433B_FMT_CS16 4
#define R433B_FMT_CS8 0x102 /* signed 8-bit IQ: converted to cu8 (+128) while loading, src/rtl_433.c:1830-1834 */
#define R433B_FMT_CF32 0x204 /* float IQ (8 bytes per sample in `data`; offsets multiples of 32): clamped and
                               scaled to cs16 on the device first, src/rtl_433.c:1811-1825; results, block size
                               and file positions are those of the cs16 stream, as in the reference */

#define R433B_FPDM_CLASSIC 0 /* FSK_PULSE_DETECT_OLD,  include/pulse_detect.h:29-34 */
#define R433B_FPDM_MINMAX 1  /* FSK_PULSE_DETECT_NEW  */
#define R433B_FPDM_AUTO 2    /* by centre frequency, src/rtl_433.c:1094-1102 */

#define R433B_PACKAGE_OOK 1 /* enum package_types, include/pulse_detect.h:23-26 */
#define R433B_PACKAGE_FSK 2

typedef struct r433b_ctx r433b_ctx;

/* Slicer-relevant part of an r_device (include/r_device.h:59-72). */
typedef struct r433b_device {
    uint32_t modulation;
    float short_width, long_width, reset_limit, gap_limit, sync_width, tolerance;
    uint32_t priority;
} r433b_device;

/* One batch of capture "files" (all of one format / rate / centre frequency).
   Stream i occupies bytes [offsets[i], offsets[i+1]) of `data`; offsets must be multiples
   of 16.  `data` is host memory (pageable or pinned) or, with data_on_device, device memory. */
typedef struct r433b_batch {
    void const *data;
    uint64_t const *offsets; /* n_streams + 1 entries, host memory */
    uint32_t n_streams;
    uint32_t sample_format;  /* R433B_FMT_* */
    uint32_t samp_rate;      /* Hz */
    uint32_t center_frequency; /* Hz */
    uint32_t fpdm_mode;      /* R433B_FPDM_* */
    uint32_t block_bytes;    /* 0 = 262144, the reference's DEFAULT_BUF_LENGTH */
    int32_t data_on_device;
    int32_t want_stages;     /* keep the AM/FM stage arrays on the device for r433b_copy_stage() */
    uint64_t const *lengths; /* optional, n_streams entries: bytes of stream i actually used (<= the gap to
                                the next offset); NULL = every stream fills its gap.  Lets files of any
                                length sit at 16-byte aligned starts. */
} r433b_batch;

/* A detected package = the integer part of pulse_data_t (include/pulse_data.h:30-50) plus
   where it was returned.  pulse/gap widths live in the pools at [pulse_off, +pulse_count). */
typedef struct r433b_package {
    uint32_t stream;
    uint32_t seq;          /* order within the stream */
    int32_t type;          /* R433B_PACKAGE_* */
    int32_t block;         /* index of the reference block that returned it; n_blocks = flush */
    uint64_t offset;
    uint64_t end_pos;      /* absolute sample index at which it was returned */
    uint32_t start_ago, end_ago, num_pulses;
    uint32_t pulse_off, pulse_count;
    int32_t ook_low_estimate, ook_high_estimate, fsk_f1_est, fsk_f2_est;
    uint32_t first_pair;   /* index of this package's device 0 in the pair table */
} r433b_package;

/* One (package, device) slicer run.  Its events are `bytes` bytes at `offset` of the event arena. */
typedef struct r433b_pair {
    uint64_t offset;
    uint32_t bytes;
    uint32_t events;       /* events stored in the arena */
    uint32_t gated_single; /* events dropped by the device's gate (r433b_set_gates): bitbuffers of one row ... */
    uint32_t gated_multi;  /* ... and of several rows */
} r433b_pair;

/* Host view of a processed batch; pointers stay valid until the next r433b_process(). */
typedef struct r433b_results {
    uint32_t n_packages;
    uint32_t n_devices;
    r433b_package const *packages; /* sorted by (stream, seq) */
    int32_t const *pulse_pool;
    int32_t const *gap_pool;
    r433b_pair const *pairs;       /* n_packages * n_devices, row = package */
    uint8_t const *events;         /* event arena */
    uint64_t event_bytes;
    uint64_t n_events;             /* events stored */
    uint64_t n_samples;            /* IQ samples consumed */
    uint64_t n_gated;              /* events counted but not stored (r433b_set_gates) */
} r433b_results;

/* Wall/device timing of the last r433b_process(), milliseconds. */
typedef struct r433b_timing {
    float h2d_ms, detect_ms, slice_ms, d2h_ms, total_ms; /* pipelined batches: kernel sums + wall total only */
    uint32_t detect_launches, slice_launches;
    float front_ms;          /* k_front (IQ -> AM), not part of detect_ms (the walk, k_detect) */
    uint32_t front_launches;
    uint32_t front_redone;   /* 64-sample chunks k_front ran twice (its guess of the filter state did not verify) */
    uint32_t front_repairs;  /* tiles whose start k_detect recomputed (k_front's guess for the tile did not fit) */
} r433b_timing;

int r433b_create(int cuda_device, r433b_ctx **out);
void r433b_destroy(r433b_ctx *ctx);
char const *r433b_last_error(r433b_ctx const *ctx);

/* pulse_detect_set_levels(), src/pulse_detect.c:86; defaults 0, 0.0, -12.1442, 9.0 (src/r_api.c:153-155) */
int r433b_set_levels(r433b_ctx *ctx, int use_mag_est, float level_limit_db, float min_level_db, float min_snr_db);
/* -Y filter / dm_state.fm_low_pass; 0 = automatic (src/r_flow.c:204) */
int r433b_set_fm_low_pass(r433b_ctx *ctx, float fm_low_pass);

/* Host-input batches are cut into `groups` runs of streams whose copy-in, kernels and copy-out
   overlap (0 = automatic, 1 = no overlap, <= 16).  Results are identical either way. */
int r433b_set_pipeline(r433b_ctx *ctx, int groups);

/* The registered decoder list in registration order (cfg->demod->r_devs, src/r_api.c:267). */
int r433b_set_devices(r433b_ctx *ctx, r433b_device const *devs, uint32_t n);
/* Same, reading the fields out of the reference's own `r_device` structs. */
struct r_device;
int r433b_set_r_devices(r433b_ctx *ctx, struct r_device *const *devs, uint32_t n);

/* Decoder length gates (SURVEY 8(f1), the dispatch fan-out of src/r_api.c:438-550 / src/pulse_slicer.c:26-66).
   Most events a slicer emits on noise are a few bits long, and every decoder turns those down with its first length
   check (DECODE_ABORT_LENGTH / _EARLY, include/r_device.h:45-53).  A gate tells the slicer kernel what that check is:
   an event with at least one row whose rows ALL hold fewer than min_bits bits is not stored; it is only counted, per
   (package, device), separately for one-row and several-row bitbuffers (many decoders test num_rows first).
   r433b_dispatch_r_devices() then books the counts exactly as account_event() would have: decode_events += n,
   decode_fails[-code] += n -- the decoders' statistics stay identical, the events never cross PCIe.  r433b_dispatch()
   does not call back for gated events (r433b_pair.gated_* has the counts).  One entry per registered device, in
   registration order; min_bits 0 = no gate.  r433b_set_devices() clears the gates.  The table for the reference's
   decoders (rtl_433_b200/data/gates_25.12.json) is derived from the decoders themselves by tools/probe_gates.py. */
typedef struct r433b_gate {
    uint16_t min_bits;
    int8_t code_single; /* decode_fn's return (0 .. -4) for a gated one-row event */
    int8_t code_multi;  /* ... for a gated event of several rows */
} r433b_gate;
int r433b_set_gates(r433b_ctx *ctx, r433b_gate const *gates, uint32_t n);

/* rtl_433 -r on every stream of the batch: block loop, flush, reset (src/rtl_433.c:1797-1854),
   then all slicers on every package.  Synchronous; results stay on the device until fetched. */
int r433b_process(r433b_ctx *ctx, r433b_batch const *batch);
/* Copy the compact results to host memory owned by the context. */
int r433b_fetch(r433b_ctx *ctx, r433b_results *out);
int r433b_get_timing(r433b_ctx const *ctx, r433b_timing *out);
/* Counters available right after r433b_process() without a fetch: packages, events stored, event bytes, samples. */
int r433b_get_counts(r433b_ctx const *ctx, uint64_t out[4]);
/* Events the gates dropped in the last batch (counted on the device). */
uint64_t r433b_get_gated(r433b_ctx const *ctx);

/* Stage arrays of one stream (batch.want_stages): what dm_state.am_buf / buf.fm held. */
int r433b_copy_stage(r433b_ctx *ctx, uint32_t stream, int16_t *am, int16_t *fm, uint64_t max_samples);

/* Position-independent 64-bit checksum (FNV-1a over 32-bit words) of everything a fetched batch holds for one
   stream: package headers, pulse / gap widths, the event bytes of every (package, device) pair.  Streams that
   carry the same samples have equal digests wherever they sit in a batch. */
int r433b_stream_digest(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, uint64_t *digest);

/* ---- host-side replay: the part of run_*_demods()/account_event() that stays on the CPU ---- */

struct bitbuffer;
struct pulse_data;

/* Re-inflate event `index` (0-based within its pair) into a caller-owned bitbuffer_t. */
int r433b_event_to_bitbuffer(uint8_t const *pair_events, uint32_t pair_bytes, uint32_t index,
        struct bitbuffer *out, uint32_t *consumed);
/* Fill a caller-owned pulse_data_t (incl. calc_rssi_snr(), src/r_flow.c:35-64) for one package. */
int r433b_package_to_pulse_data(r433b_ctx const *ctx, r433b_results const *res, uint32_t package,
        struct pulse_data *out);
/* float sample_file_pos of the block that returned the package (src/rtl_433.c:1839) */
float r433b_package_file_pos(r433b_ctx const *ctx, r433b_results const *res, uint32_t package);

/* Called once per event in the reference's order: package -> priority class -> registration
   order -> event order.  Return value is the decoder's (account_event's `ret`); > 0 in a
   priority class stops later classes of that package (src/r_api.c:444). */
typedef int (*r433b_event_fn)(void *user, uint32_t package, uint32_t device, struct pulse_data const *pd,
        struct bitbuffer *bits);
int r433b_dispatch(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, r433b_event_fn fn, void *user);
/* Same with the real r_device list: calls decode_fn and keeps the per-decoder statistics
   exactly as account_event() does (src/pulse_slicer.c:26-66). */
int r433b_dispatch_r_devices(r433b_ctx *ctx, r433b_results const *res, uint32_t stream,
        struct r_device *const *devs, uint32_t n);
/* Asynchronous batches: r433b_process() + r433b_fetch() of `batch` on a worker thread of the context.  The descriptor
   arrays are copied, the sample data must stay valid until r433b_wait().  One batch in flight per context, and the
   context must not be used until it has been waited for.  To overlap the GPU with the host replay use two contexts
   on one device alternately: submit(A, batch k+1); dispatch(results of B = batch k); wait(A); swap. */
int r433b_submit(r433b_ctx *ctx, r433b_batch const *batch);
int r433b_wait(r433b_ctx *ctx, r433b_results *out);

/* Threaded replay (SURVEY 8(f1)): stream s is replayed by worker s % n_sets, each worker calling the decoders of its
   own set of r_device instances (dev_sets[w][0 .. n_devs): registered separately, so statistics and decoder contexts
   are per worker; one instance is never entered by two threads).  Order within a stream is the reference's.  The
   caller adds up the per-set statistics.  Decoders that keep file-scope state between calls (secplus_v1/v2,
   ikea_sparsnas, arad_ms_meter in 25.12) see the streams of one worker only, in that worker's order. */
int r433b_dispatch_r_devices_parallel(r433b_ctx *ctx, r433b_results const *res, struct r_device *const *const *dev_sets,
        uint32_t n_devs, uint32_t n_sets);

/* ---- pulse analyzer (SURVEY 8(f3)): `rtl_433 -A`, src/pulse_analyzer.c:279-560, for every package of a batch ----
   The five width histograms of each package are built on the GPU (one thread per package and histogram), the guess
   of the modulation, the RfRaw rendering and the text are finished on the host from those bins, and the trial
   demodulation runs each package through the slicer of ITS guessed flex device on the GPU again. */
typedef struct r433b_hist_bin { /* hist_bin_t, src/pulse_analyzer.c:23-29 */
    uint32_t count;
    int32_t sum, mean, min, max;
} r433b_hist_bin;
typedef struct r433b_histogram { /* histogram_t, :32-35 */
    uint32_t bins_count;
    r433b_hist_bin bins[16];
} r433b_histogram;
typedef struct r433b_analysis {
    r433b_histogram hist[5]; /* as printed: pulses, gaps, pulse+gap periods, gap+pulse periods, all timings (fused) */
    int32_t total_period;    /* pulse_total_period, :289-296 */
} r433b_analysis;
typedef struct r433b_guess { /* the "Analyzer Device" the reference fills in, :355-459 */
    uint32_t modulation;     /* include/r_device.h:24-40, 0 = no clue */
    float short_width, long_width, reset_limit, gap_limit, sync_width, tolerance;
    int32_t last_gap;        /* >= 0: the package's last gap is overwritten with this before slicing (:531,:538,:545,:551) */
    int32_t sliced;          /* the reference calls a slicer for this guess */
} r433b_guess;
/* Analyze every package of the fetched batch (after r433b_fetch()). */
int r433b_analyze(r433b_ctx *ctx, r433b_results const *res);
int r433b_analysis_get(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, r433b_analysis *out, r433b_guess *guess);
/* The text pulse_analyzer() prints to stderr for the package, up to the trial demodulation's own log output
   (snprintf convention). */
size_t r433b_analysis_text(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, char *buf, size_t cap);
/* The events of the trial demodulation (compact wire format, see r433b_event_to_bitbuffer). */
int r433b_analysis_events(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, uint8_t const **events,
        uint32_t *bytes, uint32_t *n_events);

/* ---- pulse-level I/O (SURVEY 8(f4)): packages that never were IQ --------------------------------------
   `rtl_433 -r file.ook` (src/rtl_433.c:1755-1790) and RfRaw test data (-y, src/rtl_433.c:1620-1650) skip the
   demodulator and hand loaded pulse_data_t to run_ook_demods() / run_fsk_demods().  Here the loaded packages
   go to the slicer kernel; fetch / dispatch / digest work as after r433b_process().  The text formats are
   read and written on the host (no GPU needed for r433b_pulses_* and r433b_format_*). */
typedef struct r433b_pulses r433b_pulses; /* a growable set of packages, each tagged with a stream (file) index */
r433b_pulses *r433b_pulses_create(void);
void r433b_pulses_destroy(r433b_pulses *ps);
void r433b_pulses_clear(r433b_pulses *ps);
/* pulse_data_load() (src/pulse_data.c:123-181) until the text is exhausted; samp_rate = cfg->samp_rate.
   Returns the number of packages appended (>= 0) or a negative error. */
int r433b_pulses_load_ook(r433b_pulses *ps, uint32_t stream, char const *text, size_t len, uint32_t samp_rate);
/* rfraw_check() + rfraw_parse() (src/rfraw.c:67-206) of one line into a zeroed pulse_data_t: 1 package, or 0 if the
   line is not RfRaw */
int r433b_pulses_load_rfraw(r433b_pulses *ps, uint32_t stream, char const *line);
/* a caller-built pulse_data_t (fsk_f2_est != 0 selects run_fsk_demods, as in the reference) */
int r433b_pulses_add(r433b_pulses *ps, uint32_t stream, struct pulse_data const *pd);
uint32_t r433b_pulses_count(r433b_pulses const *ps);
int r433b_pulses_get(r433b_pulses const *ps, uint32_t index, struct pulse_data *out);
/* All slicers of the registered devices on every package of the set (the slicer stage only: no IQ, no detector). */
int r433b_process_pulses(r433b_ctx *ctx, r433b_pulses const *ps);

/* Writers; all return the length of the full text (snprintf convention), writing at most cap bytes.
   pulse_data_dump() src/pulse_data.c:193-226 (`received` = text after ";received ", NULL leaves the line out);
   pulse_data_print_pulse_header() :183-191; pulse_data_print_vcd() :102-121 (ch_id '\'' = AM/OOK, '"' = FM/FSK);
   pulse_data_print_vcd_header() :78-100; pulse_data_dump_raw() :58-68 (logic.u8: 0x02 OOK, 0x04 FSK). */
size_t r433b_format_ook(struct pulse_data const *pd, char const *received, char *buf, size_t cap);
size_t r433b_format_ook_header(char const *created, char *buf, size_t cap);
size_t r433b_format_vcd(struct pulse_data const *pd, int ch_id, char *buf, size_t cap);
size_t r433b_format_vcd_header(uint32_t sample_rate, char const *date, char *buf, size_t cap);
void r433b_dump_logic_u8(uint8_t *buf, uint64_t len, uint64_t buf_offset, struct pulse_data const *pd, uint8_t bits);

#ifdef __cplusplus
}
#endif
#endif /* R433B_H_ */
