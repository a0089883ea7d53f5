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

/* One batch of capture "files" (all of one format / rate / centre frequency; r433b_process_mixed takes them per stream).
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
    uint32_t idle_skipped;   /* IDLE tiles k_detect ruled out from their summaries without walking them */
    uint32_t idle_rewalks;   /* runs of such tiles walked again because their end state could not be resolved */
    float grab_ms;           /* k_grab of the last r433b_grab_copy() / r433b_grab_tail() (device time, no copy-out) */
    uint32_t chain_folds;       /* chained batches: chunk ends that folded a deferred carrier-estimate log ... */
    uint32_t chain_fm_rebuilds; /* ... and that made the FM filter state exact at the chunk end */
    float grab_ring_ms;      /* grabbing chains: k_grab_ring of the last chained batch, with the k_grab that saved the
                                ring bytes it overwrote (device time) */
    uint32_t split_segments; /* segmented replay (r433b_set_split): slots walked in pass 1, 0 when the batch ran unsplit */
    uint32_t split_rewalks;  /* segments walked again from their predecessor's end state */
    uint32_t split_rounds;   /* rewalk launches */
    float split_merge_ms;    /* k_split_merge_scan + k_split_merge (device time) */
    uint32_t mixed_classes;  /* r433b_process_mixed: detector classes of the batch (0 for every other batch) */
    float mixed_order_ms;    /* k_mixed_order: the packages regrouped by sample rate (device time) */
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

/* Segmented replay: k_detect walks one stream with one warp, so a batch of a few long captures leaves most of the GPU
   idle.  With splitting on, r433b_process() (and r433b_submit()) and r433b_process_mixed() cut each long stream at
   block boundaries into segments of segment_blocks blocks and walk them on separate warps:
   - pass 0 walks, as a file start, the warmup_blocks blocks in front of every segment but a stream's first; its end
     state is the segment's seed (the state the detector would have had the recording begun there);
   - pass 1 walks every segment, the first from the file start and every other from its seed;
   - a segment whose seed differs from its predecessor's end state (every field that can still be read: detector,
     AM and FM filters, carried IQ sample, deferred carrier-estimate log, the open package's trains) is walked again
     from that end state, in rounds, until every segment has started from the exact state;
   - the packages of every segment's last walk are merged on the device and sliced once.
   The results are those of the unsplit batch, bit for bit, whatever the seeds were.
   - segment_blocks 0 turns splitting off (the default).  R433B_SPLIT_AUTO chooses from the batch: it splits only when
     the batch has fewer streams than k_detect has resident warps (streams_per_sm x SMs, 32 x 132 on an H100), only
     streams of at least 4 segments of at least 2 blocks, with segments sized so that the slots number about one per
     resident warp.
   - warmup_blocks is 1 .. segment_blocks (R433B_EINVAL otherwise; with R433B_SPLIT_AUTO it is capped to the chosen
     segment).  A warm-up never reaches in front of its stream's start.
   - Batches with want_stages, chained batches (unless their chain opted in, see r433b_chain_split) and batches in
     which no stream has two segments run unsplit.
   - Memory on the device, per slot: the state and pulse trains of the walk and of its seed (about 40 KB), plus one
     rewalk slot per stream.  r433b_timing.split_* report what the schedule did. */
#define R433B_SPLIT_AUTO 0xffffffffu
int r433b_set_split(r433b_ctx *ctx, uint32_t segment_blocks, uint32_t warmup_blocks);

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
/* ---- mixed batches: capture files of different sample formats, rates and centre frequencies in one batch ----------
   `rtl_433 -r f1 -r f2 ...` takes its files one after another and sets the sample size, rate and FPDM at each file
   (src/rtl_433.c:1703-1745).  r433b_process_mixed() does the same for a batch whose stream i is described by fmt[i];
   the results are those of r433b_process() on each file alone, in the caller's stream order.
   - The batch's sample_format, samp_rate and center_frequency must be 0 (R433B_EINVAL otherwise).  fpdm_mode,
     block_bytes, lengths and data_on_device keep their meaning; R433B_FPDM_AUTO is resolved per stream from its centre
     frequency.  block_bytes must be a whole number of tiles for every sample size present.
   - Per stream: the rate is not 0; the offset is a multiple of 16 bytes (32 for cf32).  Without lengths the offsets
     ascend and stream i fills its gap; with lengths, stream i is [offsets[i], offsets[i] + lengths[i]), which must end by
     offsets[n_streams], and the offsets need not ascend.
   - want_stages returns R433B_EINVAL.  There is no asynchronous (r433b_submit) form; the chained form is
     r433b_process_mixed_chained() below.  Host input goes to the device in one copy, without time slices
     (r433b_set_pipeline).
   - Streams that one detector launch can walk together (the same sample size after load-time conversion, cs8 flip,
     rate and resolved FPDM) form a class.  Each class is one launch of k_front and k_detect; the launches run
     side by side on a small pool of CUDA streams.  r433b_timing: front_ms is the wall time from the first launch to
     the end of the last k_front, detect_ms from the start of the first k_detect to the end of the last; mixed_classes
     counts the classes, detect_launches the launches (a class whose streams lie in two device buffers, the caller's
     and that of the converted cf32 streams, takes one per buffer).
   - r433b_set_split applies as to r433b_process(): the segments are cut from every stream's bytes after conversion,
     in whole blocks, and R433B_SPLIT_AUTO counts the blocks of all streams.  Every pass (warm-ups, segments) and every
     rewalk round launches each class with segments in it once, side by side as above, and a round takes the first
     rejected segment of every stream of every class.  The results are those of the unsplit mixed batch, bit for bit.
     r433b_timing of a split mixed batch: split_segments, split_rewalks, split_rounds and split_merge_ms as for
     r433b_set_split; detect_launches and front_launches count the class launches of every pass and round, those of
     attempts that overflowed the arenas included; front_ms and detect_ms add up the spans above over the passes;
     mixed_classes is that of the unsplit batch; mixed_order_ms is 0 (the merge leaves the packages in rate order).
   - Afterwards everything works as after r433b_process(), and every value refers to the stream's own format, rate and
     centre frequency: fetch, digests, r433b_package_to_pulse_data(), r433b_package_file_pos(), the dispatch calls,
     the analyzer and the grabber.  The grabber's run is every stream's used bytes in the caller's order, so a window
     may reach back into an earlier file of another sample size, as the reference's does. */
typedef struct r433b_stream_format {
    uint32_t sample_format;    /* R433B_FMT_CU8 / _CS8 / _CS16 / _CF32 */
    uint32_t samp_rate;        /* Hz, != 0 */
    uint32_t center_frequency; /* Hz */
} r433b_stream_format;
int r433b_process_mixed(r433b_ctx *ctx, r433b_batch const *batch, r433b_stream_format const *fmt /* n_streams */);
/* ---- chained batches: files longer than one batch, corpora larger than memory, buffers as they arrive ----------
   The reference pushes a file through push_sdr_flow() one block at a time and carries O(1) state between the calls
   (src/rtl_433.c:1827).  A chain does the same for the streams of consecutive batches: slot i of the chain carries the
   demodulator state of one file from one r433b_process_chained() call to the next.

   The rule: cut a file into chunks at whole-block boundaries and pass them, in order, as stream i of consecutive
   chained batches.  The results equal those of the uncut file: every r433b_package field, the pulse and gap widths,
   every pair and event byte, the stage arrays (each chunk's part), the analyzer text, and the decoders' output and
   statistics.
   - Every chunk but a file's last holds a whole number of blocks: a multiple of block_bytes input bytes (2 x
     block_bytes for cf32).  Other lengths return R433B_EINVAL.
   - last[i] != 0: the file ends with this chunk (the flush runs); the slot then starts a new file, as `rtl_433 -r a
     -r b` does: its next chunk starts from the reset state with seq 0.  An empty chunk that is not the last changes
     nothing; an empty last chunk only flushes.
   - Packages report absolute offset, end_pos and block; seq continues across chunks; r433b_package_file_pos() gives
     the uncut file's sample_file_pos.  fetch, dispatch*, analyze, digests and gates work on a chained batch unchanged.
   - While any slot is inside a file, the sample format, rate, centre frequency (and so FPDM), block size, levels,
     FM low-pass and whether FM is on (which follows from the devices) must not change: R433B_ESTATE.  A batch whose
     n_streams differs from the chain's returns R433B_EINVAL.  r433b_grab_plan() and r433b_grab_tail() on a batch of
     a chain that does not grab (r433b_chain_grab below) return R433B_ESTATE.
   - A chain belongs to the context that created it and owns its device memory: per slot the carried state, the
     pulse-train scratch (19.2 KB) and a copy of both (a batch whose result arenas overflow runs again from it), about
     40 KB per slot.  r433b_destroy() frees the device memory of the context's chains; such a chain only accepts
     r433b_chain_destroy().  After a failed r433b_process_chained() the chain is undefined.
   - A chained batch walks each slot's chunk on one warp, whatever r433b_set_split says; r433b_chain_split below lets
     one chain's batches split each chunk across warps instead. */
typedef struct r433b_chain r433b_chain;
/* every slot at a file start */
int r433b_chain_create(r433b_ctx *ctx, uint32_t n_streams, r433b_chain **out);
void r433b_chain_destroy(r433b_chain *chain);
/* batch stream i is the next chunk of slot i; last[i] != 0: the file ends with it (flush, then a new file) */
int r433b_process_chained(r433b_ctx *ctx, r433b_batch const *batch, r433b_chain *chain, uint8_t const *last);
/* absolute sample index of the first sample of slot i's chunk in the last chained batch */
int r433b_chain_base(r433b_chain const *chain, uint32_t stream, uint64_t *first_sample);
/* The signal grabber on a chain (`rtl_433 -S`, see the grabber below): every slot is its own grabber run, as one
   rtl_433 process with one receiver is.  For a slot's files, taken in order, the grabs equal those of
   `rtl_433 -S <mode> -r f1 -r f2 ...`, and those of one unchained batch that holds the files in that order.
   - Opt-in, in one mode (R433B_GRAB_*) for the chain's life: a frame's decision takes in the events of every call it
     spans.  Call it while every slot is at a file start (R433B_ESTATE otherwise, and when the chain grabs already).
   - It allocates one R433B_GRAB_RING (3 MiB) ring per slot on the device, R433B_ENOMEM if that fails: 12.9 GB for
     4096 slots.  A batch of chunks longer than one block also keeps, until the next chained batch, the older ring
     bytes its append overwrote that its frames may still read: at most min(chunk, ring) - 1 block per slot.
   - A slot's run is the used bytes of its chunks in call order, across its files, after load-time conversion (cs8 as
     cu8, cf32 as cs16).  The ring is never cleared between files; ring bytes the run never wrote read as zeros.
   - Frames are tracked per slot and per file (reset_sdr_flow()) and carried from one call to the next: a frame may
     span any number of calls and end at a later block call or at its file's flush.  Its events (modes 2-3) and
     analyzer verdict (mode 4) are gathered over every call it spans.
   - After each chained batch, r433b_grab_plan(ctx, res, mode, NULL, ...) lists the grabs whose frames ended in it,
     slot by slot.  prior must be NULL and mode the chain's (R433B_EINVAL otherwise).  In r433b_grab, stream is the
     slot; counter is the grab's 1-based ordinal in its slot's run (sg_counter when no name existed: the access() loop
     is the caller's, one per slot); first_package / n_packages name the frame's packages in this batch (those of
     earlier batches are known by seq); run_end counts the slot run's bytes.  Modes 2-4 need their dispatch (and
     r433b_analyze()) per batch, as unchained.  r433b_grab_copy() then works as unchained, until the next chained
     batch; r433b_grab_tail() returns R433B_ESTATE.
   - A chained batch on a grabbing chain whose last batch was not planned returns R433B_ESTATE: its frames would be
     lost.  When appending a batch to the rings fails, the call fails and the chain's rings no longer match its runs:
     later chained batches and plans of that chain return R433B_ESTATE. */
int r433b_chain_grab(r433b_chain *chain, int mode);
/* Segmented replay for the chained batches of this chain: stream i's chunk is cut into segments of segment_blocks
   blocks (R433B_SPLIT_AUTO: chosen from the batch as r433b_set_split does), segment 0 starts from the state the chain
   carried for slot i, the others from warm-up seeds, verified and rewalked as in r433b_set_split.  Results equal the
   unsplit chain's, so it may be turned on, off (0) or changed between any two chained batches.
   - warmup_blocks is 1 .. segment_blocks (R433B_EINVAL otherwise, and for a chain whose context is gone).  Warm-ups
     lie inside the chunk: a segment near the chunk start is seeded from the chunk start, and verified like any other.
   - Batches with want_stages, and batches in which no chunk has two segments, run unsplit.  r433b_timing.split_*
     report what the schedule did.  The chain's state is written once the whole batch has succeeded, so an arena
     overflow reruns the schedule from the state the chain carried.
   - Memory on the device: that of r433b_set_split for the batch's segments, in the context. */
int r433b_chain_split(r433b_chain *chain, uint32_t segment_blocks, uint32_t warmup_blocks);
/* Mixed batches on a chain: several receivers on different bands, one slot each, or a corpus of mixed formats too large
   for the device.  Batch stream i is the next chunk of slot i's file, described by fmt[i]; for every slot the results
   are those of its files processed uncut and alone (the chain rule above, with the per-stream formats of
   r433b_process_mixed()): every r433b_package field including seq, offset, end_pos and block, the widths, pairs,
   events, analyzer text, pulse_data_t and sample_file_pos.
   - The batch's arguments are those of r433b_process_mixed(), the chain's those of r433b_process_chained(): n_streams
     equals the chain's, the chain belongs to this context, and a chunk that is not its file's last is whole blocks of
     that slot's own input (2 x block_bytes for cf32).  want_stages and a null fmt return R433B_EINVAL.
   - A slot's sample format, rate, centre frequency and resolved FPDM may change only at that slot's file start.
     block_bytes, the levels, the FM low-pass and whether FM is on are shared by the whole chain and may not change
     while any slot is inside a file.  Both return R433B_ESTATE.
   - A chain whose open files were begun by this call refuses r433b_process_chained(), and one whose open files were
     begun by r433b_process_chained() refuses this call, both with R433B_ESTATE.  While every slot is at a file start,
     either may follow.
   - A refused call leaves the context and the chain as they were.  A chain's state is written only once the whole
     batch has succeeded, so an arena overflow reruns from the state the chain carried.
   - It runs unsplit, also on a chain that opted into r433b_chain_split (r433b_timing.split_segments is 0).  There is
     no asynchronous form, and host input goes to the device in one copy per call.
   - The grabber works as on any chain (r433b_chain_grab, while every slot is at a file start): each slot is its own
     run across its files, whatever their formats, and its grabs equal those of one r433b_process_mixed() batch
     holding that slot's files in order. */
int r433b_process_mixed_chained(r433b_ctx *ctx, r433b_batch const *batch, r433b_stream_format const *fmt,
                                r433b_chain *chain, uint8_t const *last);

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
   stream: package headers, pulse / gap widths, the events of every (package, device) pair, hashed as if every
   event were stored in the long form (no one-word rows or events), with that form's byte count.  Streams that
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

/* ---- signal grabber (`rtl_433 -S all|unknown|known|undecoded`, src/samp_grab.c, src/r_flow.c:345-362) ----------
   A frame is a run of consecutive block calls of one stream that each return at least one package.  It ends at the
   first later call that returns none, or at the stream's flush; when the mode selects it, the reference writes the
   window `samp_grab_write()` cuts out of its ring of everything the run has pushed (R433B_GRAB_RING bytes, never
   cleared between files).  The run is the used bytes of every stream in batch order, after load-time conversion:
   cs8 is grabbed as cu8 (+128), cf32 as cs16.  Ring bytes the run never wrote are zero.
   r433b_grab_plan() emulates the block calls of the fetched batch and lists the files; r433b_grab_copy() gathers
   their bytes from the batch as it lies on the device (k_grab).  Batch data given with data_on_device must stay
   valid until the last r433b_grab_copy() of the batch. */
#define R433B_GRAB_ALL 1       /* grab_mode values of src/rtl_433.c:650-676 */
#define R433B_GRAB_UNKNOWN 2   /* frames whose packages no decoder decoded (needs a dispatch of every stream) */
#define R433B_GRAB_KNOWN 3     /* frames with at least one decoded message (idem) */
#define R433B_GRAB_UNDECODED 4 /* unknown frames pulse_analyzer_check() finds structure in (also needs r433b_analyze) */
#define R433B_GRAB_RING (12u * 262144u) /* SIGNAL_GRABBER_BUFFER, include/rtl_433.h:22 */

/* What the run pushed before this batch.  NULL prior = the batch starts the run (counter 1, as samp_grab_create()). */
typedef struct r433b_grab_ring {
    uint64_t pushed;      /* bytes pushed so far in the run */
    uint8_t const *tail;  /* host memory: the last min(pushed, R433B_GRAB_RING) of them */
    uint32_t counter;     /* sg_counter: the next file number to try */
} r433b_grab_ring;

/* One file samp_grab_write() writes: "g%03u_%gM_%gk.cu8" (or .cs16) with counter, center_frequency / 1e6 and
   samp_rate / 1e3.  The reference skips names that exist (access()) and counts on: that loop is the caller's, and the
   counter it ends with is the next batch's prior.counter. */
typedef struct r433b_grab {
    uint32_t stream;        /* the stream whose block call ended the frame */
    uint32_t first_package; /* index into r433b_results.packages of the frame's first package */
    uint32_t n_packages;    /* packages of the frame */
    uint32_t grab_len;      /* samples, as printed ("%u samples") */
    uint32_t bytes;         /* signal_bsize: the file's size */
    uint32_t counter;       /* prior counter + index of the grab in the batch */
    int64_t run_end;        /* run byte position at which the window ends (before wrapping in the ring) */
} r433b_grab;

/* Plan the files of the last fetched batch in `mode` (R433B_GRAB_*).  *grabs points into the context and stays valid
   until the next plan or batch.  Modes 2-4 need every stream that has packages dispatched (r433b_dispatch*: they
   record each package's p_events, the run_*_demods() return); mode 4 also needs r433b_analyze(). */
int r433b_grab_plan(r433b_ctx *ctx, r433b_results const *res, int mode, r433b_grab_ring const *prior,
        r433b_grab const **grabs, uint32_t *n);
/* The bytes of grabs [first, first + count) of the last plan back to back into `out` (host, cap bytes). */
int r433b_grab_copy(r433b_ctx *ctx, r433b_results const *res, uint32_t first, uint32_t count, uint8_t *out, size_t cap);
/* The next batch's prior: the run's byte count after this batch and its last min(pushed, R433B_GRAB_RING) bytes
   (`tail` holds R433B_GRAB_RING bytes).  The counter is the caller's (see r433b_grab). */
int r433b_grab_tail(r433b_ctx *ctx, r433b_results const *res, uint8_t *tail, uint64_t *pushed);

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
