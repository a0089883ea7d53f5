// r433b_api.cu -- the C ABI declared in include/r433b.h: context, batch processing on the GPU,
// result fetch, and the CPU-side replay that feeds events to decoders in the reference's order.
// There is no CPU implementation of the DSP here: every sample goes through k_detect/k_slice2.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <exception>
#include <atomic>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "../../include/r433b.h"
#include "../../include/r433b_abi.h"
#include "r433b_kernels.cuh"
#include "r433b_host.hpp"
#include "r433b_pulses.hpp"
#include "r433b_analyze.cuh"
#include "r433b_analyze_host.hpp"
#include "r433b_grab.cuh"
#include "r433b_split.cuh"
#include "r433b_mixed.cuh"

using namespace r433b;

// Kernel launches go through one macro so that the tests can build this translation unit against the SIMT
// emulator (tests/simt/): there the same kernels run one fibre per CUDA thread on the CPU.  The product build
// (nvcc, no R433B_SIMT_EMU) is always the <<< >>> form.
#ifdef R433B_SIMT_EMU
#define R4_LAUNCH(kernel, grid, block, smem, stream, ...) simt::launch(dim3(grid), dim3(block), (size_t)(smem), kernel, __VA_ARGS__)
#else
#define R4_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

static_assert(sizeof(struct bitbuffer) == 6604, "bitbuffer_t layout");
static_assert(sizeof(struct pulse_data) == 9672, "pulse_data_t layout");
static_assert(sizeof(struct r_device) == 152, "r_device layout");
static_assert(offsetof(struct bitbuffer, bb) == 204, "bitbuffer_t.bb offset");

namespace {

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

struct HostBuf {
    void *p = nullptr;
    size_t cap = 0;
};

// A stream's frame between block calls (src/r_flow.c:345-362): ages of its first and last package, the decoded
// events and the analyzer verdict of its packages so far.  Zero when no frame is open.
struct GrabFrame {
    uint32_t start_ago = 0, end_ago = 0, quality = 0;
    uint64_t events = 0;
};

} // namespace

struct r433b_ctx {
    int device = 0;
    std::string err;
    std::mutex err_mu; // the replay workers of r433b_dispatch_r_devices_parallel() may fail at the same time
    // detector / demod configuration
    int use_mag = 0;
    float level_limit = 0.0f, min_level = -12.1442f, min_snr = 9.0f, fm_low_pass = 0.0f;
    std::vector<r433b_device> devs;
    std::vector<r433b_gate> gates; // empty, or one per device (r433b_set_gates)
    // last batch (kept for the host replay)
    r433b_batch batch{};
    std::vector<uint64_t> offsets, lengths; // lengths[i] = bytes of stream i in use
    bool processed = false, fetched = false;
    int n_sms = 132;        // cudaDevAttrMultiProcessorCount of `device`
    int spoil_front = 0; // R433B_SPOIL_FRONT=1|2|3: k_front starts from wrong guesses (tests of the redo / repair paths)
    // R433B_TEST_CAPS=pkg,pool,arena: initial package / pulse-pool / event-arena caps in place of the defaults (0 keeps
    // a default), so that small inputs take the overflow-and-rerun paths in the tests; growth is unchanged
    size_t min_caps[3] = {0, 0, 0};
    Levels lv{};
    // device memory (grow only)
    DevBuf d_data, d_offsets, d_train, d_pkgs, d_ppool, d_gpool, d_counters, d_am, d_fm;
    DevBuf d_devparams, d_lists, d_pairs, d_arena, d_cursor;
    size_t pkg_cap = 0, pool_cap = 0, arena_cap = 0;
    unsigned n_ook = 0, n_fsk = 0;
    // counts of the last batch
    unsigned n_pkgs = 0, pool_used = 0;
    unsigned long long event_bytes = 0, n_events = 0, n_samples = 0, n_gated = 0;
    // pinned host result buffers
    HostBuf h_pkgs, h_ppool, h_gpool, h_pairs, h_events;
    r433b_timing timing{};
    cudaEvent_t ev[6]{};
    // pipelined path (host input): copy-in / detect / slice / copy-out streams and per-group events
    int pipeline_groups = 0; // 0 = automatic, 1 = off
    cudaStream_t s_in = nullptr, s_det = nullptr, s_out = nullptr;
    static constexpr int kMaxGroups = 16;
    cudaEvent_t ev_in[kMaxGroups]{}, ev_det[kMaxGroups]{}, ev_slc[kMaxGroups]{}, ev_t[4 * kMaxGroups]{}, ev_f[kMaxGroups]{}, ev_init = nullptr;
    DevBuf d_order; // k_bucket: package indices sorted by (type, length), per range
    DevBuf d_sort, d_copy; // k_bucket's tables (SortScratch) and k_slice2's lane-interleaved copy of the widths
    DevBuf d_ranges, d_state, d_lengths, d_stage, d_raw, d_log, d_amoff, d_chunks, d_tiles;
    std::vector<uint64_t> am_offsets; // first sample of stream i in d_am (multiples of the tile), n_streams + 1
    HostBuf h_ranges;
    bool d2h_done = false;
    // pulse-level input (r433b_process_pulses): per-package facts the package record has no field for;
    // r433b_package.end_pos is the index into this table
    bool pulse_mode = false;
    std::vector<PulseSet::Meta> pulse_meta;
    // pulse analyzer (r433b_analyze): results in DEVICE package order; dev_index[i] = device position of the
    // i-th package of the fetched (sorted) array
    std::vector<uint32_t> dev_index;
    bool analyzed = false;
    std::vector<r433b_analysis> an;
    std::vector<r433b_guess> an_guess;
    std::vector<std::string> an_text;
    std::vector<r433b_pair> an_pairs;
    std::vector<uint8_t> an_events;
    DevBuf d_an, d_an_dev, d_an_gap, d_an_pairs, d_an_arena;
    // r433b_submit / r433b_wait: one batch in flight on a worker thread
    std::thread worker;
    bool in_flight = false;
    int worker_rc = 0;
    r433b_batch sub_batch{};
    std::vector<uint64_t> sub_offsets, sub_lengths;
    r433b_results sub_res{};
    // signal grabber: where the batch's bytes lie on the device, what the dispatch returned per package (sorted
    // order) and per stream, the last plan and its segments
    uint8_t const *grab_src = nullptr;
    unsigned grab_flip = 0;
    std::vector<uint32_t> p_events;
    std::vector<uint8_t> dispatched;
    std::vector<r433b_grab> grabs;
    std::vector<int64_t> grab_newest; // per grab: bytes the run had pushed when the frame ended
    bool grab_planned = false;
    uint64_t grab_pushed = 0;         // run bytes before this batch (prior->pushed)
    uint64_t grab_prior_bytes = 0;    // of which the device copy of the tail holds the last ones
    std::vector<uint64_t> grab_cum;   // run offset of stream i within the batch (used bytes), n_streams + 1
    DevBuf d_grab_prior, d_grab_segs, d_grab_stage;
    // the last batch was a chained one (r433b_process_chained): absolute sample index of each stream's first sample,
    // and its chain (null once that chain is destroyed)
    bool chained = false;
    std::vector<uint64_t> chain_base;
    r433b_chain *chain_last = nullptr;
    std::vector<r433b_chain *> chains; // alive: r433b_destroy() frees their device memory and detaches them
    // segmented replay (r433b_set_split): segment / warm-up blocks (0: off), R433B_SPOIL_SEED=1 (tests of the rewalk
    // path), the slots' states and trains, their seeds, the rewalk launch's, the launch views and the merge tables
    uint32_t split_blocks = 0, split_warmup = 1;
    int spoil_seed = 0;
    DevBuf d_sp_state, d_sp_train, d_sp_seed, d_sp_seed_train, d_sp_rw_state, d_sp_rw_train;
    DevBuf d_sp_view, d_sp_flags, d_sp_list, d_sp_eq, d_sp_tab, d_sp_pkgs, d_sp_ppool, d_sp_gpool;
    // mixed batches (r433b_process_mixed): per caller stream its sample size, rate, centre frequency, and where its bytes
    // (cf32: converted to cs16) lie on the device with the flip they are read with; empty for every other batch
    struct MixedStream {
        uint32_t SS, rate, center, flip;
        uint8_t const *src;
    };
    std::vector<MixedStream> mixed;
    static constexpr int kMixedStreams = 4; // the CUDA streams the class launches go round-robin onto
    cudaStream_t s_mx[kMixedStreams]{};
    std::vector<cudaEvent_t> ev_mx;         // per launch: k_front done, k_detect done
    DevBuf d_mx_tab, d_mx_pkgs;
};

// What the carried state depends on: per slot its format, which must not change inside one of its files ...
struct SlotFormat {
    uint32_t sample_format, samp_rate, center_frequency, fpdm;
    bool operator==(SlotFormat const &o) const
    {
        return sample_format == o.sample_format && samp_rate == o.samp_rate && center_frequency == o.center_frequency
                && fpdm == o.fpdm;
    }
};

// ... and what the whole chain shares, which must not change while any of its slots has an open file
struct ChainSettings {
    uint32_t block_bytes;
    int use_mag, enable_fm;
    float level_limit, min_level, min_snr, fm_low_pass;
    bool operator==(ChainSettings const &o) const
    {
        return block_bytes == o.block_bytes && use_mag == o.use_mag && enable_fm == o.enable_fm
                && level_limit == o.level_limit && min_level == o.min_level && min_snr == o.min_snr
                && fm_low_pass == o.fm_low_pass;
    }
};

struct r433b_chain {
    r433b_ctx *ctx = nullptr;
    uint32_t n = 0;
    // device: StreamState per slot, the pulse-train scratch per slot, copies of both taken in front of every batch
    // (a batch whose result arenas overflow is run again from them), the cont / last flags and the bases of a batch
    DevBuf d_state, d_train, d_state_copy, d_train_copy, d_flags, d_base;
    std::vector<uint8_t> open;     // slot i is inside a file
    std::vector<uint64_t> next;    // ... whose next chunk starts at this absolute sample
    std::vector<uint64_t> base;    // first sample of slot i's chunk in the last chained batch
    ChainSettings settings{};
    std::vector<SlotFormat> fmt;   // per slot, of the last chained batch
    bool mixed = false;            // the last chained batch was r433b_process_mixed_chained(): so are the open files
    // segmented replay of this chain's batches (r433b_chain_split): segment / warm-up blocks, 0: off
    uint32_t split_blocks = 0, split_warmup = 1;
    // signal grabber (r433b_chain_grab): each slot is its own run with a kGrabRingBytes ring on the device
    int grab_mode = 0;
    bool grab_pending = false;     // the last chained batch has not been planned yet
    bool grab_failed = false;      // appending a batch to the rings failed: they no longer match the runs
    DevBuf d_ring, d_pre, d_ring_slots;
    std::vector<uint64_t> run;     // bytes slot i's run has pushed, after the last chained batch ...
    std::vector<uint64_t> run_c0;  // ... and before it
    // the ring bytes [pre_lo, min(run_c0, run - ring)) that the last append overwrote but whose frames may still need
    // them, saved at d_pre + pre_off
    std::vector<uint64_t> pre_lo, pre_off;
    std::vector<GrabFrame> frame, frame_next; // per slot, before the last chained batch and after it (its plan)
    std::vector<uint32_t> counter, counter_next;
    std::vector<uint8_t> ended;    // the slot's file ended with the last chained batch
};

struct r433b_pulses {
    PulseSet set;
};

namespace {
void chain_free_device(r433b_chain *ch)
{
    for (DevBuf *b : {&ch->d_state, &ch->d_train, &ch->d_state_copy, &ch->d_train_copy, &ch->d_flags, &ch->d_base,
                      &ch->d_ring, &ch->d_pre, &ch->d_ring_slots}) {
        if (b->p) cudaFree(b->p);
        b->p = nullptr;
        b->cap = 0;
    }
}
} // namespace

namespace {

int fail(r433b_ctx *c, int code, char const *what, cudaError_t e = cudaSuccess)
{
    if (c) {
        std::lock_guard<std::mutex> lock(c->err_mu);
        c->err = what;
        if (e != cudaSuccess) {
            c->err += ": ";
            c->err += cudaGetErrorString(e);
        }
    }
    return code;
}

#define CU(call)                                                   \
    do {                                                           \
        cudaError_t e_ = (call);                                   \
        if (e_ != cudaSuccess) return fail(ctx, R433B_ECUDA, #call, e_); \
    } while (0)

// cs8 is read as cu8: the load-time +128 of src/rtl_433.c:1830-1834 is an XOR of every byte's sign bit
unsigned dp_flip_of(uint32_t sample_format) { return sample_format == R433B_FMT_CS8 ? 0x80808080u : 0u; }

// What the host replay reads of a stream's format: bytes per sample (dm_state.sample_size), rate, centre frequency.  A
// mixed batch has them per stream, every other batch once.
struct StreamFormat {
    uint32_t SS, rate, center;
};
StreamFormat stream_format(r433b_ctx const *ctx, uint32_t s)
{
    if (ctx->mixed.empty()) return {ctx->batch.sample_format, ctx->batch.samp_rate, ctx->batch.center_frequency};
    r433b_ctx::MixedStream const &m = ctx->mixed[s];
    return {m.SS, m.rate, m.center};
}

int dev_reserve(r433b_ctx *ctx, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return 0;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
#ifdef R433B_EXACT_ALLOC // tests under the emulator: a buffer ends where its cap does, so a guard page behind it
                         // catches a kernel that writes even one word past the cap
    size_t want = bytes;
#else
    size_t want = bytes + bytes / 8 + 256;
#endif
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) return fail(ctx, R433B_ENOMEM, "cudaMalloc", e);
    b.cap = want;
    return 0;
}

int host_reserve(r433b_ctx *ctx, HostBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return 0;
    if (b.p) cudaFreeHost(b.p);
    b.p = nullptr;
    b.cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMallocHost(&b.p, want);
    if (e != cudaSuccess) return fail(ctx, R433B_ENOMEM, "cudaMallocHost", e);
    b.cap = want;
    return 0;
}

} // namespace

extern "C" {

int r433b_create(int cuda_device, r433b_ctx **out)
{
    if (!out) return R433B_EINVAL;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0 || cuda_device < 0 || cuda_device >= n) {
        fprintf(stderr, "r433b_create: no usable CUDA device %d (%s); there is no CPU fallback\n", cuda_device,
                e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0 or index out of range");
        return R433B_ECUDA;
    }
    r433b_ctx *ctx = new (std::nothrow) r433b_ctx();
    if (!ctx) return R433B_ENOMEM;
    ctx->device = cuda_device;
    if (cudaSetDevice(cuda_device) != cudaSuccess) {
        delete ctx;
        return R433B_ECUDA;
    }
    // both kernels live on shared memory (staged IQ tiles, AM tiles + walk state): ask for the largest carve-out
    cudaFuncSetAttribute((void const *)k_front<2>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaFuncSetAttribute((void const *)k_front<4>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaFuncSetAttribute((void const *)k_detect<2>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaFuncSetAttribute((void const *)k_detect<4>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    // k_slice2: the carve-out that holds kSliceCtasPerSm CTAs of windows (plus the 1 KiB the system reserves per CTA)
    // out of H100's 228 KiB per SM; the rest stays L1 for the pulse loads
    cudaFuncSetAttribute((void const *)k_slice2, cudaFuncAttributePreferredSharedMemoryCarveout,
                         (int)((kSliceCtasPerSm * (sizeof(g_slice_win) + sizeof(g_slice_seg) + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024)));
    for (auto &v : ctx->ev) cudaEventCreate(&v);
    cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_det, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking);
    for (auto &v : ctx->s_mx) cudaStreamCreateWithFlags(&v, cudaStreamNonBlocking);
    for (auto &v : ctx->ev_in) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_det) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_slc) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_t) cudaEventCreate(&v);
    for (auto &v : ctx->ev_f) cudaEventCreate(&v);
    cudaEventCreateWithFlags(&ctx->ev_init, cudaEventDisableTiming);
    ctx->lv = compute_levels(0, 0.0f, -12.1442f, 9.0f);
    if (char const *v = getenv("R433B_SPOIL_FRONT")) ctx->spoil_front = atoi(v);
    if (char const *v = getenv("R433B_SPOIL_SEED")) ctx->spoil_seed = atoi(v);
    if (char const *v = getenv("R433B_TEST_CAPS")) {
        unsigned long long c[3] = {0, 0, 0};
        sscanf(v, "%llu,%llu,%llu", &c[0], &c[1], &c[2]);
        for (int i = 0; i < 3; ++i) ctx->min_caps[i] = (size_t)c[i];
    }
    if (cudaDeviceGetAttribute(&ctx->n_sms, cudaDevAttrMultiProcessorCount, cuda_device) != cudaSuccess || ctx->n_sms <= 0)
        ctx->n_sms = 132;
    *out = ctx;
    return R433B_OK;
}

void r433b_destroy(r433b_ctx *ctx)
{
    if (!ctx) return;
    if (ctx->worker.joinable()) ctx->worker.join();
    cudaSetDevice(ctx->device);
    for (r433b_chain *ch : ctx->chains) { // a chain outliving its context only holds host memory from here on
        chain_free_device(ch);
        ch->ctx = nullptr;
    }
    for (DevBuf *b : {&ctx->d_data, &ctx->d_offsets, &ctx->d_train, &ctx->d_pkgs, &ctx->d_ppool, &ctx->d_gpool,
                 &ctx->d_counters, &ctx->d_am, &ctx->d_fm, &ctx->d_devparams, &ctx->d_lists, &ctx->d_pairs,
                 &ctx->d_arena, &ctx->d_cursor, &ctx->d_ranges, &ctx->d_state, &ctx->d_lengths, &ctx->d_stage, &ctx->d_raw, &ctx->d_log, &ctx->d_amoff, &ctx->d_chunks, &ctx->d_tiles,
                 &ctx->d_order, &ctx->d_sort, &ctx->d_copy, &ctx->d_an, &ctx->d_an_dev, &ctx->d_an_gap, &ctx->d_an_pairs, &ctx->d_an_arena,
                 &ctx->d_grab_prior, &ctx->d_grab_segs, &ctx->d_grab_stage, &ctx->d_sp_state, &ctx->d_sp_train,
                 &ctx->d_sp_seed, &ctx->d_sp_seed_train, &ctx->d_sp_rw_state, &ctx->d_sp_rw_train, &ctx->d_sp_view,
                 &ctx->d_sp_flags, &ctx->d_sp_list, &ctx->d_sp_eq, &ctx->d_sp_tab, &ctx->d_sp_pkgs, &ctx->d_sp_ppool,
                 &ctx->d_sp_gpool, &ctx->d_mx_tab, &ctx->d_mx_pkgs})
        if (b->p) cudaFree(b->p);
    for (HostBuf *b : {&ctx->h_pkgs, &ctx->h_ppool, &ctx->h_gpool, &ctx->h_pairs, &ctx->h_events, &ctx->h_ranges})
        if (b->p) cudaFreeHost(b->p);
    for (auto &v : ctx->ev)
        if (v) cudaEventDestroy(v);
    for (auto *arr : {ctx->ev_in, ctx->ev_det, ctx->ev_slc})
        for (int i = 0; i < r433b_ctx::kMaxGroups; ++i)
            if (arr[i]) cudaEventDestroy(arr[i]);
    for (auto &v : ctx->ev_t)
        if (v) cudaEventDestroy(v);
    for (auto &v : ctx->ev_f)
        if (v) cudaEventDestroy(v);
    if (ctx->ev_init) cudaEventDestroy(ctx->ev_init);
    for (auto &v : ctx->ev_mx) cudaEventDestroy(v);
    for (cudaStream_t st : {ctx->s_in, ctx->s_det, ctx->s_out})
        if (st) cudaStreamDestroy(st);
    for (cudaStream_t st : ctx->s_mx)
        if (st) cudaStreamDestroy(st);
    delete ctx;
}

char const *r433b_last_error(r433b_ctx const *ctx) { return ctx ? ctx->err.c_str() : "no context"; }

int r433b_set_levels(r433b_ctx *ctx, int use_mag_est, float level_limit_db, float min_level_db, float min_snr_db)
{
    if (!ctx) return R433B_EINVAL;
    ctx->use_mag = use_mag_est ? 1 : 0;
    ctx->level_limit = level_limit_db;
    ctx->min_level = min_level_db;
    ctx->min_snr = min_snr_db;
    ctx->lv = compute_levels(ctx->use_mag, level_limit_db, min_level_db, min_snr_db);
    return R433B_OK;
}

int r433b_set_fm_low_pass(r433b_ctx *ctx, float v)
{
    if (!ctx) return R433B_EINVAL;
    ctx->fm_low_pass = v;
    return R433B_OK;
}

int r433b_set_pipeline(r433b_ctx *ctx, int groups)
{
    if (!ctx || groups < 0 || groups > r433b_ctx::kMaxGroups) return R433B_EINVAL;
    ctx->pipeline_groups = groups;
    return R433B_OK;
}

int r433b_set_split(r433b_ctx *ctx, uint32_t segment_blocks, uint32_t warmup_blocks)
{
    if (!ctx) return R433B_EINVAL;
    if (segment_blocks && (warmup_blocks < 1 || (segment_blocks != R433B_SPLIT_AUTO && warmup_blocks > segment_blocks)))
        return fail(ctx, R433B_EINVAL, "r433b_set_split: warmup_blocks must be 1 .. segment_blocks");
    ctx->split_blocks = segment_blocks;
    ctx->split_warmup = segment_blocks ? warmup_blocks : 1;
    return R433B_OK;
}

int r433b_chain_split(r433b_chain *chain, uint32_t segment_blocks, uint32_t warmup_blocks)
{
    if (!chain || !chain->ctx) return R433B_EINVAL;
    if (segment_blocks && (warmup_blocks < 1 || (segment_blocks != R433B_SPLIT_AUTO && warmup_blocks > segment_blocks)))
        return fail(chain->ctx, R433B_EINVAL, "r433b_chain_split: warmup_blocks must be 1 .. segment_blocks");
    chain->split_blocks = segment_blocks;
    chain->split_warmup = segment_blocks ? warmup_blocks : 1;
    return R433B_OK;
}

int r433b_set_devices(r433b_ctx *ctx, r433b_device const *devs, uint32_t n)
{
    if (!ctx || (n && !devs)) return R433B_EINVAL;
    ctx->devs.assign(devs, devs + n);
    ctx->gates.clear();
    return R433B_OK;
}

int r433b_set_gates(r433b_ctx *ctx, r433b_gate const *gates, uint32_t n)
{
    if (!ctx || (n && !gates)) return R433B_EINVAL;
    if (n && n != ctx->devs.size()) return fail(ctx, R433B_EINVAL, "r433b_set_gates: one gate per registered device");
    for (uint32_t i = 0; i < n; ++i)
        if (gates[i].code_single > 0 || gates[i].code_single < -4 || gates[i].code_multi > 0 || gates[i].code_multi < -4)
            return fail(ctx, R433B_EINVAL, "r433b_set_gates: codes are decode_fn returns 0 .. -4");
    ctx->gates.assign(gates, gates + n);
    return R433B_OK;
}

uint64_t r433b_get_gated(r433b_ctx const *ctx) { return ctx && ctx->processed ? ctx->n_gated : 0; }

int r433b_set_r_devices(r433b_ctx *ctx, struct r_device *const *devs, uint32_t n)
{
    if (!ctx || (n && !devs)) return R433B_EINVAL;
    ctx->devs.resize(n);
    ctx->gates.clear();
    for (uint32_t i = 0; i < n; ++i) {
        struct r_device const *d = devs[i];
        r433b_device &o = ctx->devs[i];
        o.modulation = d->modulation;
        o.short_width = d->short_width;
        o.long_width = d->long_width;
        o.reset_limit = d->reset_limit;
        o.gap_limit = d->gap_limit;
        o.sync_width = d->sync_width;
        o.tolerance = d->tolerance;
        o.priority = d->priority;
    }
    return R433B_OK;
}

namespace {

// The slicer tables of a batch: every device scaled to each sample rate of `rates` (with its gate; the package
// range of rate g reads entries [g * n_devs, (g + 1) * n_devs)) and the OOK / FSK device lists.  Also sizes
// k_slice2's staging scratch: the kernel runs as a fixed grid whose warps fetch work items (GroupRange::next), and
// every thread of that grid owns kStageWords of scratch for the staged single pass.
int upload_slicer_tables(r433b_ctx *ctx, std::vector<uint32_t> const &rates, cudaStream_t st)
{
    size_t const n_devs = ctx->devs.size();
    std::vector<SlicerParams> sp(rates.size() * n_devs);
    for (size_t g = 0; g < rates.size(); ++g)
        for (size_t i = 0; i < n_devs; ++i) {
            sp[g * n_devs + i] = scale_device(ctx->devs[i], rates[g]);
            if (!ctx->gates.empty()) sp[g * n_devs + i].gate = ctx->gates[i].min_bits;
        }
    std::vector<unsigned> lists = slice_list(ctx->devs, 1), fsk = slice_list(ctx->devs, 2);
    ctx->n_ook = (unsigned)lists.size();
    ctx->n_fsk = (unsigned)fsk.size();
    lists.insert(lists.end(), fsk.begin(), fsk.end());
    if (int r = dev_reserve(ctx, ctx->d_devparams, std::max<size_t>(1, sp.size()) * sizeof(SlicerParams))) return r;
    if (int r = dev_reserve(ctx, ctx->d_lists, (lists.size() + 1) * sizeof(unsigned))) return r;
    size_t const stage_threads = (size_t)ctx->n_sms * kSliceCtasPerSm * kSliceThreads;
    if (int r = dev_reserve(ctx, ctx->d_stage, stage_threads * kStageWords * sizeof(uint32_t))) return r;
    if (!sp.empty()) CU(cudaMemcpyAsync(ctx->d_devparams.p, sp.data(), sp.size() * sizeof(SlicerParams), cudaMemcpyHostToDevice, st));
    if (!lists.empty()) CU(cudaMemcpyAsync(ctx->d_lists.p, lists.data(), lists.size() * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    return R433B_OK;
}

// k_bucket's tables and k_slice2's copy of the widths for ranges of at most `pkgs` packages and `pool_entries` pool
// entries, reserved next to the pools.  The copy of a range is at most its pool entries plus one group of the
// longest package per type (r433b_kernels.cuh), so it cannot overflow for the packages the detector stored.  The
// slice launches of a batch all run on one stream, one range after the other: one copy serves every range.
int reserve_sort(r433b_ctx *ctx, size_t pkgs, size_t pool_entries, cudaStream_t st)
{
    size_t const cap0 = ctx->d_sort.cap;
    if (int r = dev_reserve(ctx, ctx->d_sort, (4 * kLenBins + pkgs / 32 + 3) * sizeof(unsigned))) return r;
    // k_bucket_count's histogram starts at zero, and every k_bucket_scan leaves it so
    if (ctx->d_sort.cap != cap0) CU(cudaMemsetAsync(ctx->d_sort.p, 0, 2 * kLenBins * sizeof(unsigned), st));
    return dev_reserve(ctx, ctx->d_copy, (pool_entries + 2 * 32 * (size_t)kMaxPulses) * sizeof(PulseGap));
}

// The slicers over one package range: k_bucket sorts its packages, k_slice2 runs every slicer on them with the
// tables of sample rate `rate_index`.  `n_pkgs` bounds the range, whose end may only be known on the device.
void launch_slice(r433b_ctx *ctx, GroupRange *range, unsigned n_pkgs, unsigned rate_index, cudaStream_t st)
{
    SortScratch ss;
    ss.hist = (unsigned *)ctx->d_sort.p;
    ss.fill = ss.hist + 2 * kLenBins;
    ss.base = ss.fill + 2 * kLenBins;
    ss.copy = (PulseGap *)ctx->d_copy.p;
    ss.copy_cap = std::min<size_t>(ctx->d_copy.cap / sizeof(PulseGap), 0xffffffffu);
    unsigned const n_devs = (unsigned)ctx->devs.size();
    r433b_package *pkgs = (r433b_package *)ctx->d_pkgs.p;
    SliceParams q{};
    q.pkgs = pkgs;
    q.range = range;
    q.order = (unsigned const *)ctx->d_order.p;
    q.copy = ss.copy;
    q.group_base = ss.base;
    q.dev = (SlicerParams const *)ctx->d_devparams.p + (size_t)rate_index * n_devs;
    q.n_devs = n_devs;
    q.ook_list = (unsigned const *)ctx->d_lists.p;
    q.fsk_list = q.ook_list + ctx->n_ook;
    q.n_ook = ctx->n_ook;
    q.n_fsk = ctx->n_fsk;
    q.pairs = (r433b_pair *)ctx->d_pairs.p;
    q.arena = (uint8_t *)ctx->d_arena.p;
    q.arena_cap = ctx->arena_cap;
    q.cursor = (SliceCursor *)ctx->d_cursor.p;
    q.stage = (uint32_t *)ctx->d_stage.p;
    unsigned const bgrid = (unsigned)ctx->n_sms * 2;
    R4_LAUNCH(k_bucket_count, bgrid, kBucketThreads, 0, st, range, pkgs, n_pkgs, n_devs, ss.hist);
    R4_LAUNCH(k_bucket_scan, 1, 32, 0, st, range, ss);
    R4_LAUNCH(k_bucket_scatter, bgrid, kBucketThreads, 0, st, range, (r433b_package const *)pkgs, n_pkgs, (unsigned *)ctx->d_order.p, ss,
              (int const *)ctx->d_ppool.p, (int const *)ctx->d_gpool.p);
    R4_LAUNCH(k_slice2, (unsigned)ctx->n_sms * kSliceCtasPerSm, kSliceThreads, 0, st, q);
}

// The slicer stage over package ranges known on the host: range g (pkg_begin / pkg_end set, the rest zero) uses
// slicer table g; the ranges hold `pool_entries` pool entries in all.  Runs again with an event arena grown to what
// the device counted until every event fits, times the stage with ev[2] -> ev[3] and leaves the event totals in the
// context.
int slice_ranges(r433b_ctx *ctx, std::vector<GroupRange> const &ranges, unsigned n_pkgs, size_t pool_entries, cudaStream_t st)
{
    unsigned const n_devs = (unsigned)ctx->devs.size();
    SliceCursor cur{};
    ctx->timing.slice_launches = 0;
    CU(cudaEventRecord(ctx->ev[2], st));
    if (n_pkgs && n_devs) {
        size_t const pair_bytes = (size_t)n_pkgs * n_devs * sizeof(r433b_pair);
        if (int r = dev_reserve(ctx, ctx->d_pairs, pair_bytes)) return r;
        if (int r = dev_reserve(ctx, ctx->d_order, (size_t)n_pkgs * sizeof(unsigned))) return r;
        if (int r = reserve_sort(ctx, n_pkgs, pool_entries, st)) return r;
        if (int r = dev_reserve(ctx, ctx->d_ranges, ranges.size() * sizeof(GroupRange))) return r;
        if (int r = dev_reserve(ctx, ctx->d_cursor, 64)) return r;
        for (int attempt = 0; attempt < 3; ++attempt) {
            if (int r = dev_reserve(ctx, ctx->d_arena, ctx->arena_cap)) return r;
            CU(cudaMemsetAsync(ctx->d_pairs.p, 0, pair_bytes, st));
            CU(cudaMemsetAsync(ctx->d_cursor.p, 0, 64, st));
            CU(cudaMemcpyAsync(ctx->d_ranges.p, ranges.data(), ranges.size() * sizeof(GroupRange), cudaMemcpyHostToDevice, st));
            for (size_t g = 0; g < ranges.size(); ++g) {
                launch_slice(ctx, (GroupRange *)ctx->d_ranges.p + g, n_pkgs, (unsigned)g, st);
                CU(cudaGetLastError());
                ctx->timing.slice_launches++;
            }
            CU(cudaMemcpyAsync(&cur, ctx->d_cursor.p, sizeof(cur), cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            if (!cur.overflow) break;
            ctx->arena_cap = (size_t)cur.bytes + (1u << 20);
            if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "event arena overflow");
        }
    }
    CU(cudaEventRecord(ctx->ev[3], st));
    CU(cudaEventSynchronize(ctx->ev[3]));
    cudaEventElapsedTime(&ctx->timing.slice_ms, ctx->ev[2], ctx->ev[3]);
    ctx->event_bytes = cur.bytes;
    ctx->n_events = cur.events;
    ctx->n_gated = cur.gated;
    return R433B_OK;
}

int chain_grab_append(r433b_ctx *ctx, r433b_chain *ch);

// What process_iq() derives from a batch's arguments
struct Shape {
    bool cf32;       // cf32 becomes cs16 on the device before anything else (src/rtl_433.c:1811-1825): from there on
    unsigned in_div; // offsets, lengths and byte counts are those of the cs16 stream (the input's / in_div)
    int SS;          // bytes per IQ sample; cs8 is cu8 after the load-time +128
    SlotFormat fmt;  // every stream's
    ChainSettings settings;
    uint64_t total_bytes, used_bytes, max_samples; // the last two of the lengths in use (adopt_batch)
};

// A chained batch's chain arguments: slot i's format fmt[i] and input bytes in_bytes[i]; `mixed`: the batch is
// r433b_process_mixed_chained()'s.  Changes nothing in the context but the error string.
int check_chain(r433b_ctx *ctx, r433b_batch const *b, r433b_chain const *ch, uint8_t const *last,
        ChainSettings const &settings, bool mixed, std::vector<SlotFormat> const &fmt, std::vector<uint64_t> const &in_bytes)
{
    std::string const who = mixed ? "r433b_process_mixed_chained: " : "r433b_process_chained: ";
    auto refuse = [&](int code, char const *what) { return fail(ctx, code, (who + what).c_str()); };
    if (ch->ctx != ctx || !last) return refuse(R433B_EINVAL, "chain of another context, or no last[]");
    if (b->n_streams != ch->n) return refuse(R433B_EINVAL, "n_streams differs from the chain's");
    if (ch->grab_failed) return refuse(R433B_ESTATE, "a batch of this grabbing chain failed while appending to its rings");
    if (ch->grab_pending)
        return refuse(R433B_ESTATE, "the grabbing chain's last batch was not planned (r433b_grab_plan): its frames would "
                                    "be lost");
    bool const open = std::find(ch->open.begin(), ch->open.end(), 1) != ch->open.end();
    if (open && ch->mixed != mixed)
        return refuse(R433B_ESTATE, mixed ? "the chain's open files were begun by r433b_process_chained"
                                          : "the chain's open files were begun by r433b_process_mixed_chained");
    bool changed = open && !(settings == ch->settings);
    for (uint32_t i = 0; i < b->n_streams && !changed; ++i) changed = ch->open[i] && !(fmt[i] == ch->fmt[i]);
    if (changed)
        return refuse(R433B_ESTATE, "format, rate, frequency, block size, levels or FM settings changed while a file of "
                                    "the chain is open");
    // a chunk that the file goes on behind is whole blocks: the next one starts on a block boundary
    for (uint32_t i = 0; i < b->n_streams; ++i) {
        uint64_t const in_div = fmt[i].sample_format == R433B_FMT_CF32 ? 2 : 1;
        if (!last[i] && in_bytes[i] % ((uint64_t)settings.block_bytes * in_div))
            return refuse(R433B_EINVAL, "a chunk that is not its file's last must be whole blocks (block_bytes, 2 x "
                                        "block_bytes of cf32 input)");
    }
    return R433B_OK;
}

// The batch's arguments, and the chain's if it has one.  Changes nothing in the context but the error string.
int check_batch(r433b_ctx *ctx, r433b_batch const *b, r433b_chain const *ch, uint8_t const *last, Shape &s)
{
    if (!ctx || !b || !b->offsets || (b->n_streams && !b->data)) return fail(ctx, R433B_EINVAL, "null argument");
    if (b->sample_format != R433B_FMT_CU8 && b->sample_format != R433B_FMT_CS16 && b->sample_format != R433B_FMT_CS8
            && b->sample_format != R433B_FMT_CF32)
        return fail(ctx, R433B_EINVAL, "sample_format must be R433B_FMT_CU8, _CS8, _CS16 or _CF32");
    s.cf32 = b->sample_format == R433B_FMT_CF32;
    s.in_div = s.cf32 ? 2 : 1;
    if (b->samp_rate == 0) return fail(ctx, R433B_EINVAL, "samp_rate is 0");
    s.SS = (int)(b->sample_format & 0xff);
    uint32_t const block_bytes = b->block_bytes ? b->block_bytes : 262144u;
    if (block_bytes % (uint32_t)(kTile * s.SS) != 0) return fail(ctx, R433B_EINVAL, "block_bytes must be a multiple of 2048 samples (4096 bytes of cu8, 8192 of cs16)");
    for (uint32_t i = 0; i <= b->n_streams; ++i) {
        if (b->offsets[i] % (16 * s.in_div)) return fail(ctx, R433B_EINVAL, "stream offsets must be multiples of 16 bytes (32 for cf32)");
        if (i && b->offsets[i] < b->offsets[i - 1]) return fail(ctx, R433B_EINVAL, "offsets not ascending");
    }
    s.total_bytes = b->n_streams ? b->offsets[b->n_streams] / s.in_div : 0;
    int enable_fm = 0;
    for (auto const &d : ctx->devs)
        if (d.modulation >= 16) enable_fm = 1;
    // src/rtl_433.c:1094-1102 and :1515-1522
    unsigned const fpdm = b->fpdm_mode == R433B_FPDM_AUTO ? (b->center_frequency > 800000000u ? 1u : 0u) : b->fpdm_mode;
    s.fmt = SlotFormat{b->sample_format, b->samp_rate, b->center_frequency, fpdm};
    s.settings = ChainSettings{block_bytes, ctx->use_mag, enable_fm, ctx->level_limit, ctx->min_level, ctx->min_snr,
                               ctx->fm_low_pass};
    if (!ch) return R433B_OK;
    std::vector<uint64_t> in_bytes(b->n_streams);
    for (uint32_t i = 0; i < b->n_streams; ++i) in_bytes[i] = b->lengths ? b->lengths[i] : b->offsets[i + 1] - b->offsets[i];
    return check_chain(ctx, b, ch, last, s.settings, false, std::vector<SlotFormat>(b->n_streams, s.fmt), in_bytes);
}

// The batch becomes the context's last one (the host replay reads it), and the results of the one before are gone
int adopt_batch(r433b_ctx *ctx, r433b_batch const *b, Shape &s)
{
    ctx->processed = ctx->fetched = false;
    ctx->chained = ctx->pulse_mode = false;
    ctx->chain_last = nullptr;
    ctx->mixed.clear();
    ctx->batch = *b;
    ctx->batch.sample_format = (uint32_t)s.SS; // the host replay only needs the sample size (dm_state.sample_size)
    ctx->batch.block_bytes = s.settings.block_bytes;
    ctx->offsets.assign(b->offsets, b->offsets + b->n_streams + 1);
    for (auto &v : ctx->offsets) v /= s.in_div;
    ctx->batch.offsets = ctx->offsets.data();
    ctx->lengths.resize(b->n_streams);
    s.used_bytes = s.max_samples = 0;
    for (uint32_t i = 0; i < b->n_streams; ++i) {
        uint64_t gap = b->offsets[i + 1] - b->offsets[i];
        ctx->lengths[i] = b->lengths ? b->lengths[i] : gap;
        if (ctx->lengths[i] > gap) return fail(ctx, R433B_EINVAL, "lengths[i] exceeds the gap to the next offset");
        if (s.cf32) ctx->lengths[i] = ctx->lengths[i] / 8 * 4; // whole IQ pairs of floats -> cs16 bytes
        s.used_bytes += ctx->lengths[i];
        s.max_samples = std::max<uint64_t>(s.max_samples, ctx->lengths[i] / s.SS);
    }
    ctx->batch.lengths = ctx->lengths.data();
    ctx->grabs.clear();
    ctx->grab_planned = false;
    ctx->timing.grab_ms = ctx->timing.grab_ring_ms = 0;
    ctx->d2h_done = false;
    return R433B_OK;
}

// The FM low-pass of a launch from its sample size, rate, FPDM and whether FM is on
void set_fm_filter(r433b_ctx const *ctx, int SS, DetectParams &dp)
{
    dp.wrap_free = 1;
    if (dp.enable_fm) {
        float lp = ctx->fm_low_pass != 0.0f ? ctx->fm_low_pass : dp.fpdm ? 0.2f : 0.1f; // src/r_flow.c:204
        fm_coeffs(SS == 4, dp.rate, lp, dp.fm_a1, dp.fm_b0);
        long long unity = SS == 2 ? 16384ll : (1ll << 30);
        dp.wrap_free = dp.fm_a1 >= 0 && dp.fm_b0 >= 0 && (long long)dp.fm_a1 + 2ll * dp.fm_b0 <= unity;
    }
}

// The device buffers of the batch (no data moved yet) and the detector's launch parameters, into a zeroed `dp`
int prepare_detect(r433b_ctx *ctx, r433b_batch const *b, Shape const &s, DetectParams &dp)
{
    int const SS = s.SS, T = kTile;
    uint8_t const *d_in = (uint8_t const *)b->data;
    if (!b->data_on_device || s.cf32) {
        if (int r = dev_reserve(ctx, ctx->d_data, s.total_bytes + 64)) return r;
        d_in = (uint8_t const *)ctx->d_data.p;
    }
    ctx->grab_src = d_in; // cf32 is grabbed as the cs16 it was converted to
    ctx->grab_flip = dp_flip_of(b->sample_format);
    if (s.cf32 && !b->data_on_device)
        if (int r = dev_reserve(ctx, ctx->d_raw, 2 * s.total_bytes + 64)) return r;
    if (int r = dev_reserve(ctx, ctx->d_offsets, (b->n_streams + 1) * sizeof(uint64_t))) return r;
    CU(cudaMemcpy(ctx->d_offsets.p, ctx->offsets.data(), (b->n_streams + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (int r = dev_reserve(ctx, ctx->d_lengths, std::max<size_t>(1, b->n_streams) * sizeof(uint64_t))) return r;
    if (b->n_streams) CU(cudaMemcpy(ctx->d_lengths.p, ctx->lengths.data(), b->n_streams * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (int r = dev_reserve(ctx, ctx->d_train, (size_t)std::max(1u, b->n_streams) * kTrainInts * sizeof(int))) return r;
    if (int r = dev_reserve(ctx, ctx->d_log, (size_t)std::max(1u, b->n_streams) * kLogCap * 2 * sizeof(unsigned))) return r;
    if (int r = dev_reserve(ctx, ctx->d_counters, 64)) return r;
    if (int r = dev_reserve(ctx, ctx->d_cursor, 64)) return r;
    // k_front's output: 16-bit AM of every sample, every stream padded to whole tiles, + the bounds of every chunk
    ctx->am_offsets.resize(b->n_streams + 1);
    ctx->am_offsets[0] = 0;
    for (uint32_t i = 0; i < b->n_streams; ++i)
        ctx->am_offsets[i + 1] = ctx->am_offsets[i] + (ctx->lengths[i] / SS + T - 1) / T * T;
    uint64_t const am_samples = ctx->am_offsets[b->n_streams];
    if (int r = dev_reserve(ctx, ctx->d_am, am_samples * sizeof(int16_t) + 16)) return r;
    if (int r = dev_reserve(ctx, ctx->d_chunks, am_samples / kChunk * sizeof(ChunkInfo) + 16)) return r;
    if (int r = dev_reserve(ctx, ctx->d_tiles, am_samples / T * sizeof(TileInfo) + 16)) return r;
    if (int r = dev_reserve(ctx, ctx->d_amoff, (b->n_streams + 1) * sizeof(uint64_t))) return r;
    CU(cudaMemcpy(ctx->d_amoff.p, ctx->am_offsets.data(), (b->n_streams + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (b->want_stages)
        if (int r = dev_reserve(ctx, ctx->d_fm, s.total_bytes / SS * sizeof(int16_t) + 16)) return r;

    dp.data = d_in;
    dp.offsets = (unsigned long long const *)ctx->d_offsets.p;
    dp.lengths = (unsigned long long const *)ctx->d_lengths.p;
    dp.n_streams = dp.stream_end = b->n_streams;
    dp.sample_end = ~0ull;
    dp.first_chunk = 1;
    dp.use_mag = ctx->use_mag;
    dp.flip = dp_flip_of(b->sample_format);
    dp.enable_fm = s.settings.enable_fm;
    dp.fpdm = (int)s.fmt.fpdm;
    dp.rate = b->samp_rate;
    dp.block_samples = s.settings.block_bytes / SS;
    dp.lv = ctx->lv;
    dp.lpf_a1 = ((int)(0.85408 * 32768)) >> 1; // src/baseband.c:151-152
    dp.lpf_b0 = ((int)(0.07296 * 32768)) >> 1;
    set_fm_filter(ctx, SS, dp);
    dp.train_scratch = (int *)ctx->d_train.p;
    dp.log_scratch = (unsigned *)ctx->d_log.p;
    dp.counters = (DetectCounters *)ctx->d_counters.p;
    dp.am_offsets = (unsigned long long const *)ctx->d_amoff.p;
    dp.am = (int16_t *)ctx->d_am.p;
    dp.chunks = (ChunkInfo const *)ctx->d_chunks.p;
    dp.tile_info = (TileInfo const *)ctx->d_tiles.p;
    dp.fm_out = b->want_stages ? (int16_t *)ctx->d_fm.p : nullptr;
    return R433B_OK;
}

int bind_detector_arenas(r433b_ctx *ctx, DetectParams &dp)
{
    if (int r = dev_reserve(ctx, ctx->d_pkgs, ctx->pkg_cap * sizeof(r433b_package))) return r;
    if (int r = dev_reserve(ctx, ctx->d_ppool, ctx->pool_cap * sizeof(int))) return r;
    if (int r = dev_reserve(ctx, ctx->d_gpool, ctx->pool_cap * sizeof(int))) return r;
    dp.pkgs = (r433b_package *)ctx->d_pkgs.p;
    dp.pkg_cap = (unsigned)std::min<size_t>(ctx->pkg_cap, 0xffffffffu);
    dp.pulse_pool = (int *)ctx->d_ppool.p;
    dp.gap_pool = (int *)ctx->d_gpool.p;
    dp.pool_cap = (unsigned)std::min<size_t>(ctx->pool_cap, 0xffffffffu);
    return R433B_OK;
}

// A chained batch: the chain's state and pulse trains, which slots continue a file, which files end, where each chunk
// lies in its file (chain_base, in slot order).  The state is copied first, so that a run that has to be repeated
// starts from it again.  A mixed batch (`order`: the slot of internal stream j) walks its streams in internal order: the
// flags and bases go to the device permuted, and the walk uses the copies, into which the caller gathers the state
// (k_split_chain_in) at every attempt; the chain's own state is written only once the batch has succeeded.
int chain_begin(r433b_ctx *ctx, r433b_chain *ch, uint8_t const *last, DetectParams &dp,
        std::vector<uint32_t> const *order = nullptr)
{
    if (!ch) return R433B_OK;
    size_t const n = ch->n;
    std::vector<uint8_t> flags(2 * n);
    std::vector<uint64_t> base(n);
    ctx->chain_base.resize(n);
    for (size_t i = 0; i < n; ++i) ctx->chain_base[i] = ch->open[i] ? ch->next[i] : 0;
    for (size_t j = 0; j < n; ++j) {
        size_t const i = order ? (*order)[j] : j;
        flags[j] = ch->open[i];
        flags[n + j] = last[i] ? 1 : 0;
        base[j] = ctx->chain_base[i];
    }
    CU(cudaMemcpy(ch->d_flags.p, flags.data(), 2 * n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ch->d_base.p, base.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    dp.cont = (unsigned char const *)ch->d_flags.p;
    dp.last = (unsigned char const *)ch->d_flags.p + n;
    dp.base = (unsigned long long const *)ch->d_base.p;
    if (order) {
        dp.state = (StreamState *)ch->d_state_copy.p;
        dp.train_scratch = (int *)ch->d_train_copy.p;
        return R433B_OK;
    }
    CU(cudaMemcpyAsync(ch->d_state_copy.p, ch->d_state.p, n * sizeof(StreamState), cudaMemcpyDeviceToDevice, 0));
    CU(cudaMemcpyAsync(ch->d_train_copy.p, ch->d_train.p, n * kTrainInts * sizeof(int), cudaMemcpyDeviceToDevice, 0));
    dp.state = (StreamState *)ch->d_state.p;
    dp.train_scratch = (int *)ch->d_train.p;
    return R433B_OK;
}

// The batch has succeeded: the chain moves on, and a grabbing chain appends the chunks to its rings (once, also after a
// run that was repeated).  fmt: every slot's format.
int chain_finish(r433b_ctx *ctx, r433b_chain *ch, uint8_t const *last, ChainSettings const &settings,
        std::vector<SlotFormat> const &fmt, bool mixed)
{
    if (!ch) return R433B_OK;
    for (uint32_t i = 0; i < ch->n; ++i) {
        ch->open[i] = last[i] ? 0 : 1;
        ch->next[i] = last[i] ? 0 : ctx->chain_base[i] + ctx->lengths[i] / stream_format(ctx, i).SS;
    }
    ch->base = ctx->chain_base;
    ch->settings = settings;
    ch->fmt = fmt;
    ch->mixed = mixed;
    ctx->chained = true;
    ctx->chain_last = ch;
    if (!ch->grab_mode) return R433B_OK;
    for (uint32_t i = 0; i < ch->n; ++i) ch->ended[i] = last[i] ? 1 : 0;
    return chain_grab_append(ctx, ch);
}

// k_front over the tiles [sample_begin, sample_end) of the streams [stream0, stream_end), then the walk over the same range
void launch_detect(r433b_ctx *ctx, DetectParams const &q, Shape const &s, cudaStream_t st, cudaEvent_t after_front)
{
    int const SS = s.SS, T = kTile;
    unsigned const n_launch = q.stream_end - q.stream0;
    uint64_t const t_end = (std::min<uint64_t>(q.sample_end, s.max_samples) + T - 1) / T, t_begin = q.sample_begin / T;
    if (t_end > t_begin) {
        FrontParams fp{};
        fp.data = q.data;
        fp.offsets = q.offsets + q.stream0;
        fp.lengths = q.lengths ? q.lengths + q.stream0 : nullptr;
        fp.am_offsets = q.am_offsets + q.stream0;
        fp.n_streams = n_launch;
        fp.tile_begin = t_begin;
        fp.tiles = (unsigned)(t_end - t_begin);
        fp.use_mag = q.use_mag;
        fp.flip = q.flip;
        fp.block_samples = q.block_samples;
        fp.a1 = q.lpf_a1;
        fp.b0 = q.lpf_b0;
        fp.am = q.am;
        fp.chunks = (ChunkInfo *)ctx->d_chunks.p;
        fp.tile_info = (TileInfo *)ctx->d_tiles.p;
        fp.counters = q.counters;
        fp.spoil = ctx->spoil_front;
        fp.state = q.state ? q.state + q.stream0 : nullptr;
        fp.cont = q.first_chunk && q.cont ? q.cont + q.stream0 : nullptr;
        uint64_t const warps = (uint64_t)n_launch * fp.tiles;
        unsigned const fgrid = (unsigned)((warps + kFrontWarps - 1) / kFrontWarps);
        void (*ffn)(FrontParams) = SS == 2 ? k_front<2> : k_front<4>;
        size_t const fsm = (size_t)kFrontWarps * (SS == 2 ? FrontStage<2>::kBytes : FrontStage<4>::kBytes);
        R4_LAUNCH(ffn, fgrid, kFrontWarps * 32, fsm, st, fp);
    }
    cudaEventRecord(after_front, st);
    unsigned grid = (n_launch + kDetectWarps - 1) / kDetectWarps;
    size_t sm = (size_t)kDetectWarps * sizeof(WarpSmem);
    void (*kfn)(DetectParams) = SS == 2 ? k_detect<2> : k_detect<4>;
    R4_LAUNCH(kfn, grid, kDetectWarps * 32, sm, st, q);
}

int check_pair_index(r433b_ctx *ctx, uint64_t n_pkgs)
{
    if (n_pkgs * ctx->devs.size() <= 0xffffffffull) return R433B_OK;
    return fail(ctx, R433B_EOVERFLOW, "packages x devices exceeds the 32-bit pair index (r433b_package.first_pair)");
}

// The result arrays of a range (packages, both pools, pairs, events): buffers and the bytes [lo, hi) of the range
struct ResultPart { HostBuf &h; DevBuf const &d; size_t lo, hi; };
std::array<ResultPart, 5> result_parts(r433b_ctx *ctx, GroupRange const &r)
{
    size_t const pk = sizeof(r433b_package), pair = ctx->devs.size() * sizeof(r433b_pair);
    return {{{ctx->h_pkgs, ctx->d_pkgs, r.pkg_begin * pk, r.pkg_end * pk},
             {ctx->h_ppool, ctx->d_ppool, r.pool_begin * sizeof(int), r.pool_end * sizeof(int)},
             {ctx->h_gpool, ctx->d_gpool, r.pool_begin * sizeof(int), r.pool_end * sizeof(int)},
             {ctx->h_pairs, ctx->d_pairs, r.pkg_begin * pair, r.pkg_end * pair},
             {ctx->h_events, ctx->d_arena, r.arena_begin, r.arena_end}}};
}

// Device to host: the results of a range, at the same offsets in the pinned buffers
int copy_results(r433b_ctx *ctx, GroupRange const &r, cudaStream_t st)
{
    for (ResultPart const &p : result_parts(ctx, r))
        if (p.hi > p.lo && p.d.p) CU(cudaMemcpyAsync((char *)p.h.p + p.lo, (char const *)p.d.p + p.lo, p.hi - p.lo, cudaMemcpyDeviceToHost, st));
    return R433B_OK;
}

// How many time slices the batch is cut into (1: one launch), of how many samples per stream.  Slices take host input
// on a uniform stride, one strided copy each; the streams' LENGTHS may differ: the kernels stop at every stream's end.
int time_slices(r433b_ctx const *ctx, r433b_batch const *b, Shape const &s, uint64_t &slice_samples)
{
    int G = ctx->pipeline_groups;
    uint64_t stride = b->n_streams ? ctx->offsets[1] - ctx->offsets[0] : 0;
    bool uniform = b->n_streams > 0 && stride > 0;
    for (uint32_t i = 0; uniform && i < b->n_streams; ++i)
        if (ctx->offsets[i + 1] - ctx->offsets[i] != stride) uniform = false;
    if (G == 0) { // slice size (tools/e2e_sweep.py sweeps it): many slices of >= 128 KiB per stream for cu8 (4096 streams);
                  // cs16 batches (1024 x 4 MiB, FM on: every launch pays the slowest stream's bursts) want >= 512 KiB
        uint64_t const min_slice = s.SS == 4 ? (512u << 10) : (128u << 10);
        G = (s.total_bytes >= (256ull << 20) && stride >= (1u << 20)) ? (int)std::min<uint64_t>(r433b_ctx::kMaxGroups, stride / min_slice) : 1;
    }
    if (b->data_on_device && ctx->pipeline_groups == 0) G = 1; // device input: slices only when asked for
    // stage arrays: k_detect's stage pass makes FM of whole streams, so that batch must be one launch
    if (b->want_stages || ctx->devs.empty() || !uniform || s.cf32) G = 1;
    slice_samples = 0;
    if (G > 1) {
        uint64_t n_samp = stride / s.SS;
        uint64_t unit = (uint64_t)kTile; // slices only have to be tile aligned: block effects use absolute positions
        slice_samples = (n_samp / G + unit - 1) / unit * unit;
        if (slice_samples == 0 || slice_samples >= n_samp) G = 1;
        else G = (int)((n_samp + slice_samples - 1) / slice_samples);
        if (G > r433b_ctx::kMaxGroups) G = 1;
    }
    return G;
}

// The time-sliced schedule: the copy-in of slice k+1 and the copy-out of finished ranges overlap the kernels of slice
// k (three streams).  detect(k) and slice(k) stay on ONE stream: both are issue-bound, running them concurrently only
// makes each slower (measured).  (Cutting by streams instead does not help: a warp needs the same wall time for its
// stream however few other warps run.)  Detector / filter state is carried between launches in `StreamState`; results
// are identical to one launch.  kFellBack: an arena overflowed; the caps have grown, the batch runs again in one launch.
constexpr int kFellBack = 1;
int run_time_sliced(r433b_ctx *ctx, r433b_batch const *b, Shape const &s, int G, uint64_t slice_samples, DetectParams &dp, DetectCounters &cnt)
{
    using clk = std::chrono::steady_clock;
    auto t_wall0 = clk::now();
    int const SS = s.SS;
    uint32_t const n_devs = (uint32_t)ctx->devs.size();
    uint64_t const stride = ctx->offsets[1] - ctx->offsets[0];
    if (int r = bind_detector_arenas(ctx, dp)) return r;
    if (int r = dev_reserve(ctx, ctx->d_order, ctx->pkg_cap * sizeof(unsigned))) return r;
    if (int r = reserve_sort(ctx, ctx->pkg_cap, ctx->pool_cap, ctx->s_det)) return r;
    size_t const pair_cap_bytes = ctx->pkg_cap * n_devs * sizeof(r433b_pair);
    if (int r = dev_reserve(ctx, ctx->d_pairs, pair_cap_bytes)) return r;
    if (int r = dev_reserve(ctx, ctx->d_arena, ctx->arena_cap)) return r;
    if (int r = dev_reserve(ctx, ctx->d_ranges, G * sizeof(GroupRange))) return r;
    if (int r = dev_reserve(ctx, ctx->d_state, (size_t)b->n_streams * sizeof(StreamState))) return r;
    if (int r = host_reserve(ctx, ctx->h_ranges, G * sizeof(GroupRange))) return r;
    if (!dp.state) dp.state = (StreamState *)ctx->d_state.p; // a chain carries its own
    GroupRange *d_rg = (GroupRange *)ctx->d_ranges.p, *h_rg = (GroupRange *)ctx->h_ranges.p;
    DetectCounters const *d_cnt = (DetectCounters const *)ctx->d_counters.p;
    SliceCursor const *d_cur = (SliceCursor const *)ctx->d_cursor.p;

    // the table uploads went through the legacy stream from pageable memory: their DMA may still be in flight when
    // cudaMemcpy returns, and s_det does not synchronise with stream 0 by itself
    CU(cudaEventRecord(ctx->ev_init, 0));
    CU(cudaStreamWaitEvent(ctx->s_det, ctx->ev_init, 0));
    CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, ctx->s_det));
    CU(cudaMemsetAsync(ctx->d_cursor.p, 0, 64, ctx->s_det));
    CU(cudaMemsetAsync(ctx->d_pairs.p, 0, pair_cap_bytes, ctx->s_det));
    CU(cudaEventRecord(ctx->ev_init, ctx->s_det));
    for (int g = 0; g < G; ++g) {
        uint64_t c0 = (uint64_t)g * slice_samples * SS, c1 = std::min<uint64_t>(stride, c0 + slice_samples * SS);
        // one strided copy: the same byte range of every stream
        if (!b->data_on_device)
            CU(cudaMemcpy2DAsync((uint8_t *)ctx->d_data.p + ctx->offsets[0] + c0, stride,
                    (uint8_t const *)b->data + ctx->offsets[0] + c0, stride, c1 - c0, b->n_streams,
                    cudaMemcpyHostToDevice, ctx->s_in));
        CU(cudaEventRecord(ctx->ev_in[g], ctx->s_in));
        CU(cudaStreamWaitEvent(ctx->s_det, ctx->ev_in[g], 0));
        R4_LAUNCH(k_mark, 1, 1, 0, ctx->s_det, d_rg + g, 0, d_cnt, d_cur);
        CU(cudaEventRecord(ctx->ev_t[4 * g + 0], ctx->s_det));
        DetectParams dg = dp;
        dg.sample_begin = (uint64_t)g * slice_samples;
        dg.sample_end = g == G - 1 ? ~0ull : (uint64_t)(g + 1) * slice_samples;
        dg.first_chunk = g == 0;
        launch_detect(ctx, dg, s, ctx->s_det, ctx->ev_f[g]);
        CU(cudaEventRecord(ctx->ev_t[4 * g + 1], ctx->s_det));
        R4_LAUNCH(k_mark, 1, 1, 0, ctx->s_det, d_rg + g, 1, d_cnt, d_cur);
        CU(cudaEventRecord(ctx->ev_det[g], ctx->s_det));
        R4_LAUNCH(k_mark, 1, 1, 0, ctx->s_det, d_rg + g, 2, d_cnt, d_cur);
        CU(cudaEventRecord(ctx->ev_t[4 * g + 2], ctx->s_det));
        launch_slice(ctx, d_rg + g, dp.pkg_cap, 0, ctx->s_det);
        CU(cudaEventRecord(ctx->ev_t[4 * g + 3], ctx->s_det));
        R4_LAUNCH(k_mark, 1, 1, 0, ctx->s_det, d_rg + g, 3, d_cnt, d_cur);
        CU(cudaMemcpyAsync(h_rg + g, d_rg + g, sizeof(GroupRange), cudaMemcpyDeviceToHost, ctx->s_det));
        CU(cudaEventRecord(ctx->ev_slc[g], ctx->s_det));
    }
    CU(cudaGetLastError());
    // copy-out of finished groups while later ones compute; only into host buffers that are
    // already large enough (they are after the first batch of a given shape)
    bool overflow = false, d2h_ok = !b->data_on_device; // device input: results stay put until r433b_fetch()
    for (int g = 0; g < G; ++g) {
        CU(cudaEventSynchronize(ctx->ev_slc[g]));
        GroupRange const r = h_rg[g];
        if (r.overflow) overflow = true;
        if (overflow) continue;
        // the same sizes r433b_fetch() reserves (+16): a buffer that passes here is never reallocated there
        for (ResultPart const &p : result_parts(ctx, r)) d2h_ok = d2h_ok && p.h.cap >= p.hi + 16;
        if (!d2h_ok) continue;
        if (int rc = copy_results(ctx, r, ctx->s_out)) return rc;
    }
    CU(cudaStreamSynchronize(ctx->s_out));
    CU(cudaMemcpy(&cnt, ctx->d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost));
    if (overflow) { // grow from what the device counted
        SliceCursor cur;
        CU(cudaMemcpy(&cur, ctx->d_cursor.p, sizeof(cur), cudaMemcpyDeviceToHost));
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)cnt.pkgs * 2 + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)cnt.pool * 2 + 4096);
        ctx->arena_cap = std::max<size_t>(ctx->arena_cap, (size_t)cur.bytes * 2 + (1u << 20));
        return kFellBack;
    }
    GroupRange const end = h_rg[G - 1];
    if (int r = check_pair_index(ctx, end.pkg_end)) return r;
    ctx->n_pkgs = end.pkg_end;
    ctx->pool_used = end.pool_end;
    ctx->event_bytes = end.arena_end;
    ctx->n_events = end.events_end;
    ctx->n_gated = end.gated_end;
    ctx->d2h_done = d2h_ok;
    auto ms = [](cudaEvent_t a, cudaEvent_t b) { float t = 0; cudaEventElapsedTime(&t, a, b); return t; };
    ctx->timing.front_ms = ctx->timing.detect_ms = ctx->timing.slice_ms = 0;
    for (int g = 0; g < G; ++g) {
        ctx->timing.front_ms += ms(ctx->ev_t[4 * g + 0], ctx->ev_f[g]);
        ctx->timing.detect_ms += ms(ctx->ev_f[g], ctx->ev_t[4 * g + 1]);
        ctx->timing.slice_ms += ms(ctx->ev_t[4 * g + 2], ctx->ev_t[4 * g + 3]);
    }
    ctx->timing.h2d_ms = 0; // overlapped: only the wall total is meaningful
    ctx->timing.total_ms = std::chrono::duration<float, std::milli>(clk::now() - t_wall0).count();
    ctx->timing.detect_launches = (unsigned)G;
    ctx->timing.slice_launches = (unsigned)G;
    return R433B_OK;
}

// The batch's samples to the device whole: host input copied, cf32 converted to cs16
int copy_in(r433b_ctx *ctx, r433b_batch const *b, Shape const &s, cudaStream_t st)
{
    if (s.cf32 && s.total_bytes) {
        void const *raw = b->data;
        if (!b->data_on_device) {
            CU(cudaMemcpyAsync(ctx->d_raw.p, b->data, 2 * s.total_bytes, cudaMemcpyHostToDevice, st));
            raw = ctx->d_raw.p;
        }
        size_t n4 = (size_t)(2 * s.total_bytes / 16); // groups of four floats (offsets are multiples of 32 bytes)
        R4_LAUNCH(k_cf32_to_cs16, ctx->n_sms * 8, 256, 0, st, (float4 const *)raw, (uint2 *)ctx->d_data.p, n4);
        CU(cudaGetLastError());
    } else if (!b->data_on_device && s.total_bytes)
        CU(cudaMemcpyAsync(ctx->d_data.p, b->data, s.total_bytes, cudaMemcpyHostToDevice, st));
    return R433B_OK;
}

// The one-launch schedule on stream 0: copy-in, the detector (again with the arenas grown to what it counted while
// they overflow), then the slicers over all its packages.  `rerun`: the detector has run on this batch before.
int run_sequential(r433b_ctx *ctx, r433b_batch const *b, Shape const &s, DetectParams &dp, r433b_chain *ch, bool rerun, DetectCounters &cnt)
{
    cudaStream_t const st = 0;
    CU(cudaEventRecord(ctx->ev[0], st));
    if (int r = copy_in(ctx, b, s, st)) return r;
    CU(cudaEventRecord(ctx->ev[1], st));

    unsigned detect_launches = 0;
    for (int attempt = 0; attempt < 3; ++attempt) {
        if (ch && (attempt > 0 || rerun)) { // from the state chain_begin() found
            CU(cudaMemcpyAsync(ch->d_state.p, ch->d_state_copy.p, ch->n * sizeof(StreamState), cudaMemcpyDeviceToDevice, st));
            CU(cudaMemcpyAsync(ch->d_train.p, ch->d_train_copy.p, ch->n * kTrainInts * sizeof(int), cudaMemcpyDeviceToDevice, st));
        }
        if (int r = bind_detector_arenas(ctx, dp)) return r;
        CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, st));
        if (b->n_streams) {
            launch_detect(ctx, dp, s, st, ctx->ev[4]);
            CU(cudaGetLastError());
            detect_launches++;
        }
        CU(cudaMemcpyAsync(&cnt, ctx->d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (!cnt.overflow) break;
        // arenas were too small: the counters hold the true need
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)cnt.pkgs + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)cnt.pool + 4096);
        if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "package arena overflow");
    }
    if (int r = check_pair_index(ctx, cnt.pkgs)) return r;
    ctx->n_pkgs = cnt.pkgs;
    ctx->pool_used = cnt.pool;
    GroupRange all{};
    all.pkg_end = ctx->n_pkgs;
    if (int r = slice_ranges(ctx, std::vector<GroupRange>{all}, ctx->n_pkgs, ctx->pool_used, st)) return r;
    cudaEventElapsedTime(&ctx->timing.h2d_ms, ctx->ev[0], ctx->ev[1]);
    ctx->timing.front_ms = 0;
    if (detect_launches) cudaEventElapsedTime(&ctx->timing.front_ms, ctx->ev[1], ctx->ev[4]);
    cudaEventElapsedTime(&ctx->timing.detect_ms, ctx->ev[detect_launches ? 4 : 1], ctx->ev[2]); // with the counter read-back
    cudaEventElapsedTime(&ctx->timing.total_ms, ctx->ev[0], ctx->ev[3]);
    ctx->timing.detect_launches = detect_launches;
    return R433B_OK;
}

// ---- detector launches per class (DESIGN §7d) -----------------------------------------------------------------------

// A class: the streams one detector launch can walk together, and the device buffer they lie in (bufs[buf] of the
// launch).  A mixed batch's internal order sorts its streams by class, stable in the caller's; a class is the streams
// [begin, end) of a launch view.  A one-format batch is one class.
struct MixedClass {
    uint32_t rate, SS, flip, fpdm, buf;
    uint32_t begin, end;
    uint64_t max_samples;
    bool same(MixedClass const &o) const
    {
        return rate == o.rate && SS == o.SS && flip == o.flip && fpdm == o.fpdm && buf == o.buf;
    }
};

// The classes of a batch over its streams in internal order, the two device buffers they read (the caller's, the cf32
// conversion region), and the first internal stream of every sample rate's slot, + n_streams: k_slice2's ranges
struct ClassSet {
    std::vector<MixedClass> classes;
    uint8_t const *bufs[2];
    std::vector<uint32_t> rate_first;
};

float elapsed_ms(cudaEvent_t a, cudaEvent_t b)
{
    float t = 0;
    cudaEventElapsedTime(&t, a, b);
    return t;
}

// One k_front + k_detect launch per class over the launch view in `dp`, each with its class's buffer, format and FM
// filter, round-robin on the CUDA stream pool behind everything stream 0 has queued; stream 0 waits for every launch.
// ev[4]: the start; ev_mx[2c] / ev_mx[2c + 1]: class c's k_front / k_detect done.
int launch_classes(r433b_ctx *ctx, DetectParams const &dp, std::vector<MixedClass> const &classes,
        uint8_t const *const bufs[2], uint32_t block_bytes)
{
    cudaStream_t const st = 0;
    while (ctx->ev_mx.size() < 2 * classes.size()) {
        cudaEvent_t e;
        CU(cudaEventCreate(&e));
        ctx->ev_mx.push_back(e);
    }
    CU(cudaEventRecord(ctx->ev[4], st));
    for (size_t c = 0; c < classes.size(); ++c) {
        MixedClass const &k = classes[c];
        cudaStream_t const ps = ctx->s_mx[c % r433b_ctx::kMixedStreams];
        DetectParams q = dp;
        q.data = bufs[k.buf];
        q.stream0 = k.begin;
        q.stream_end = k.end;
        q.flip = k.flip;
        q.fpdm = (int)k.fpdm;
        q.rate = k.rate;
        q.block_samples = block_bytes / k.SS;
        set_fm_filter(ctx, (int)k.SS, q);
        Shape sh{};
        sh.SS = (int)k.SS;
        sh.max_samples = k.max_samples;
        CU(cudaStreamWaitEvent(ps, ctx->ev[4], 0));
        launch_detect(ctx, q, sh, ps, ctx->ev_mx[2 * c]);
        CU(cudaGetLastError());
        CU(cudaEventRecord(ctx->ev_mx[2 * c + 1], ps));
        CU(cudaStreamWaitEvent(st, ctx->ev_mx[2 * c + 1], 0));
    }
    return R433B_OK;
}

// The spans of the last launch_classes() of `n` classes, once it has completed: k_front from the start to the last
// class's k_front end, k_detect from the first class's k_detect start to the last one's end
void class_spans(r433b_ctx const *ctx, size_t n, float &front_ms, float &detect_ms)
{
    float front_end = 0, detect_begin = 0, detect_end = 0;
    for (size_t c = 0; c < n; ++c) {
        float const f = elapsed_ms(ctx->ev[4], ctx->ev_mx[2 * c]), d = elapsed_ms(ctx->ev[4], ctx->ev_mx[2 * c + 1]);
        front_end = std::max(front_end, f);
        detect_begin = c ? std::min(detect_begin, f) : f;
        detect_end = std::max(detect_end, d);
    }
    front_ms = front_end;
    detect_ms = detect_end - detect_begin;
}

// ---- segmented replay (r433b_set_split, DESIGN §7c) ---------------------------------------------------------------

// The segments of a batch, stream by stream: segment k is bytes [begin, begin + bytes) of batch stream `stream`
struct SplitPlan {
    std::vector<uint32_t> stream, first; // first: the stream's first segment
    std::vector<uint64_t> begin, bytes;
    uint64_t warmup = 1;                 // blocks
};

// Segments of segment_blocks blocks (R433B_SPLIT_AUTO: chosen from the batch) behind warm-ups of warmup_blocks, cut from
// each stream's used bytes (a chained batch's: each slot's chunk), stream by stream in `order` (a mixed batch's internal
// order; null: the batch's).  false: the batch runs unsplit (splitting off, stage arrays, or no stream of two segments).
bool plan_split(r433b_ctx const *ctx, r433b_batch const *b, Shape const &s, uint32_t segment_blocks, uint32_t warmup_blocks,
        SplitPlan &p, std::vector<uint32_t> const *order = nullptr)
{
    if (!segment_blocks || b->want_stages || !b->n_streams) return false;
    uint64_t const bb = s.settings.block_bytes;
    uint64_t seg = segment_blocks, min_blocks = 0;
    if (segment_blocks == R433B_SPLIT_AUTO) {
        uint64_t const warps = (uint64_t)ctx->n_sms * kDetectCtasPerSm * kDetectWarps, n = b->n_streams;
        if (n >= warps) return false;
        uint64_t blocks = 0;
        for (uint64_t i = 0; i < n; ++i) blocks += (ctx->lengths[i] + bb - 1) / bb;
        seg = std::max<uint64_t>(kSplitMinSegmentBlocks, (blocks + warps - 1) / warps);
        min_blocks = seg * kSplitMinSegments;
    }
    p.warmup = std::min<uint64_t>(warmup_blocks, seg);
    bool any = false;
    for (uint32_t j = 0; j < b->n_streams; ++j) {
        uint32_t const i = order ? (*order)[j] : j;
        uint64_t const len = ctx->lengths[i], blocks = (len + bb - 1) / bb;
        uint32_t const first = (uint32_t)p.stream.size();
        bool const split = blocks > seg && blocks >= min_blocks;
        any = any || split;
        for (uint64_t b0 = 0; b0 == 0 || (split && b0 < blocks); b0 += seg) {
            p.stream.push_back(i);
            p.first.push_back(first);
            p.begin.push_back(b0 * bb);
            p.bytes.push_back(split ? std::min(len, (b0 + seg) * bb) - b0 * bb : len);
        }
    }
    return any;
}

// The streams of one pass of the split schedule: stream i walks bytes [off, off + len) of its class's buffer as a
// chained chunk whose sample 0 is absolute sample `base` of its file, from the state it holds where `cont`, flushing
// where `last`.  `cls`: its class; the streams of a class are consecutive.
struct SplitLaunch {
    std::vector<uint64_t> off, len, base;
    std::vector<uint8_t> cont, last;
    std::vector<uint32_t> cls;
    void add(uint64_t o, uint64_t l, uint64_t b0, bool c, bool e, uint32_t k)
    {
        off.push_back(o);
        len.push_back(l);
        base.push_back(b0);
        cont.push_back(c ? 1 : 0);
        last.push_back(e ? 1 : 0);
        cls.push_back(k);
    }
};

// What the passes of a split batch add up: class launches, the k_front and k_detect spans
struct SplitTotals {
    unsigned launches = 0;
    float front_ms = 0, detect_ms = 0;
};

// One pass: its view to the device, then k_front and k_detect per class with streams in it (launch_classes) with
// `state` / `train` as their chain state; the counters are read back into `cnt` (they go on from the pass before)
int split_launch(r433b_ctx *ctx, DetectParams const &dp, Shape const &s, ClassSet const &cs, SplitLaunch const &v,
        StreamState *state, int *train, DetectCounters &cnt, SplitTotals &tot)
{
    cudaStream_t const st = 0;
    size_t const n = v.off.size();
    if (!n) return R433B_OK;
    std::vector<uint64_t> view(4 * n + 2); // offsets (n + 1), lengths, AM offsets (n + 1), bases
    uint64_t *off = view.data(), *len = off + n + 1, *amoff = len + n, *base = amoff + n + 1;
    std::vector<MixedClass> runs; // the pass's class launches: the view's runs of one class
    amoff[0] = 0;
    for (size_t i = 0; i < n; ++i) {
        MixedClass const &k = cs.classes[v.cls[i]];
        if (i == 0 || v.cls[i] != v.cls[i - 1]) {
            runs.push_back(k);
            runs.back().begin = (uint32_t)i;
            runs.back().max_samples = 0;
        }
        runs.back().end = (uint32_t)i + 1;
        runs.back().max_samples = std::max<uint64_t>(runs.back().max_samples, v.len[i] / k.SS);
        off[i] = v.off[i];
        len[i] = v.len[i];
        base[i] = v.base[i];
        amoff[i + 1] = amoff[i] + (v.len[i] / k.SS + kTile - 1) / kTile * kTile;
    }
    off[n] = s.total_bytes;
    std::vector<uint8_t> flags(v.cont);
    flags.insert(flags.end(), v.last.begin(), v.last.end());
    CU(cudaMemcpyAsync(ctx->d_sp_view.p, view.data(), view.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_sp_flags.p, flags.data(), flags.size(), cudaMemcpyHostToDevice, st));
    auto const *d_view = (unsigned long long const *)ctx->d_sp_view.p;
    DetectParams q = dp;
    q.offsets = d_view;
    q.lengths = d_view + n + 1;
    q.am_offsets = d_view + 2 * n + 1;
    q.base = d_view + 3 * n + 2;
    q.cont = (unsigned char const *)ctx->d_sp_flags.p;
    q.last = q.cont + n;
    q.n_streams = q.stream_end = (unsigned)n;
    q.state = state;
    q.train_scratch = train;
    q.fm_out = nullptr;
    if (int r = launch_classes(ctx, q, runs, cs.bufs, s.settings.block_bytes)) return r;
    CU(cudaMemcpyAsync(&cnt, ctx->d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    float f = 0, d = 0;
    class_spans(ctx, runs.size(), f, d);
    tot.front_ms += f;
    tot.detect_ms += d;
    tot.launches += (unsigned)runs.size();
    return R433B_OK;
}

// k_split_compare over the listed segments; eq[k] = its seed equals its predecessor's end state
int split_compare(r433b_ctx *ctx, std::vector<uint32_t> const &segs, std::vector<uint8_t> &eq)
{
    cudaStream_t const st = 0;
    unsigned const m = (unsigned)segs.size();
    if (!m) return R433B_OK;
    size_t const n = eq.size();
    unsigned *list = (unsigned *)ctx->d_sp_list.p;
    std::vector<uint8_t> got(m);
    CU(cudaMemcpyAsync(list, segs.data(), m * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    R4_LAUNCH(k_split_compare, (m + kSplitWarps - 1) / kSplitWarps, kSplitWarps * 32, 0, st,
              (StreamState const *)ctx->d_sp_seed.p, (int const *)ctx->d_sp_seed_train.p, (StreamState const *)ctx->d_sp_state.p,
              (int const *)ctx->d_sp_train.p, (unsigned const *)list, m, (unsigned char *)ctx->d_sp_eq.p, list + n);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(got.data(), ctx->d_sp_eq.p, m, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (unsigned i = 0; i < m; ++i) eq[segs[i]] = got[i];
    return R433B_OK;
}

// The split schedule on stream 0, behind the copy-in: pass 0 (warm-ups -> seeds), pass 1 (every segment), rounds of
// rewalks until every segment has started from its predecessor's exact end state, the merge, then the slicers over the
// merged packages, one range per sample rate.  Every pass and round launches each class with segments in it once
// (`cs`; the plan is in the classes' internal order), so a round takes the first rejected segment of every stream of
// every class.  An arena overflow in any pass grows the caps from what the device counted and runs the schedule again
// from pass 0.  With a chain, stream i's segments lie at the chain's base for slot i, the first starts from the state
// the chain carried (loaded in front of pass 1, so a rerun loads it again), the last ends as the chunk does (last[i]),
// and the chain takes the last's end state once everything has succeeded.
int run_split(r433b_ctx *ctx, r433b_batch const *b, Shape const &s, SplitPlan const &p, ClassSet const &cs,
        DetectParams const &dp0, r433b_chain *ch, uint8_t const *last_chunk, DetectCounters &cnt)
{
    cudaStream_t const st = 0;
    size_t const n = p.stream.size(), ns = b->n_streams, tr = (size_t)kTrainInts * sizeof(int);
    uint64_t const bb = s.settings.block_bytes;
    for (auto [buf, bytes] : {std::pair<DevBuf *, size_t>{&ctx->d_sp_state, n * sizeof(StreamState)}, {&ctx->d_sp_train, n * tr},
                              {&ctx->d_sp_seed, n * sizeof(StreamState)}, {&ctx->d_sp_seed_train, n * tr},
                              {&ctx->d_sp_rw_state, ns * sizeof(StreamState)}, {&ctx->d_sp_rw_train, ns * tr},
                              {&ctx->d_log, n * kLogCap * 2 * sizeof(unsigned)}, {&ctx->d_sp_view, (4 * n + 2) * sizeof(uint64_t)},
                              {&ctx->d_sp_flags, 2 * n}, {&ctx->d_sp_list, (3 * n + 2 + 2 * ns) * sizeof(unsigned)},
                              {&ctx->d_sp_eq, n}})
        if (int r = dev_reserve(ctx, *buf, bytes)) return r;
    StreamState *const state = (StreamState *)ctx->d_sp_state.p, *const rw_state = (StreamState *)ctx->d_sp_rw_state.p;
    int *const train = (int *)ctx->d_sp_train.p, *const rw_train = (int *)ctx->d_sp_rw_train.p;
    unsigned *const list = (unsigned *)ctx->d_sp_list.p, *const start_seq = list + n, *const pkg_base = start_seq + n;
    unsigned *const slot_first = pkg_base + n + 2, *const slot_last = slot_first + ns; // per stream: its first / last segment
    DetectParams dp = dp0;
    dp.log_scratch = (unsigned *)ctx->d_log.p;

    // pass 0 walks the warm-up in front of every segment but a stream's first (those slots walk nothing), pass 1 the
    // segments; slot k is segment k in both
    SplitLaunch warm, walk;
    std::vector<uint32_t> later, slots(2 * ns); // every segment but a stream's first; each stream's first and last
    std::vector<uint32_t> stream_seg;           // the first segment of internal stream j, + n
    for (size_t k = 0, c = 0; k < n; ++k) {
        uint32_t const i = p.stream[k];
        bool const first = p.first[k] == k, last = k + 1 == n || p.first[k + 1] != p.first[k];
        if (first) stream_seg.push_back((uint32_t)k);
        while (cs.classes[c].end < stream_seg.size()) ++c;
        uint64_t const SS = cs.classes[c].SS;
        uint64_t const o = ctx->offsets[i], w0 = first || p.begin[k] < p.warmup * bb ? 0 : p.begin[k] - p.warmup * bb;
        uint64_t const base = ch ? ctx->chain_base[i] : 0;
        warm.add(o + w0, first ? 0 : p.begin[k] - w0, base + w0 / SS, false, false, (uint32_t)c);
        walk.add(o + p.begin[k], p.bytes[k], base + p.begin[k] / SS, first ? ch && ch->open[i] : true,
                 last && (!ch || last_chunk[i]), (uint32_t)c);
        if (!first) later.push_back((uint32_t)k);
        if (first) slots[i] = (uint32_t)k;
        if (last) slots[ns + i] = (uint32_t)k;
    }
    stream_seg.push_back((uint32_t)n);
    if (ch) CU(cudaMemcpyAsync(slot_first, slots.data(), 2 * ns * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    SplitTotals tot;
    unsigned rewalks = 0, rounds = 0;
    DetectCounters warm_cnt{};
    std::vector<uint32_t> final_walk, launch_lo, map_off, seg_of;
    for (int attempt = 0;; ++attempt) {
        if (int r = bind_detector_arenas(ctx, dp)) return r;
        CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, st));
        if (int r = split_launch(ctx, dp, s, cs, warm, state, train, warm_cnt, tot)) return r;
        // the warm-ups' packages are not kept: the arenas start again behind them
        CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, st));
        CU(cudaMemcpyAsync(ctx->d_sp_seed.p, state, n * sizeof(StreamState), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(ctx->d_sp_seed_train.p, train, n * tr, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemsetAsync(start_seq, 0, n * sizeof(unsigned), st));
        if (ch) {
            R4_LAUNCH(k_split_chain_in, (unsigned)((ns + kSplitWarps - 1) / kSplitWarps), kSplitWarps * 32, 0, st,
                      (StreamState const *)ch->d_state.p, (int const *)ch->d_train.p, (unsigned char const *)ch->d_flags.p,
                      (unsigned const *)slot_first, (unsigned)ns, state, train, start_seq);
            CU(cudaGetLastError());
        }
        if (ctx->spoil_seed) { // only the copy that is compared: pass 1 starts from the seeds as they were
            R4_LAUNCH(k_split_spoil, (unsigned)((n + 127) / 128), 128, 0, st, (StreamState *)ctx->d_sp_seed.p,
                      (int *)ctx->d_sp_seed_train.p, (unsigned)n);
            CU(cudaGetLastError());
        }
        if (int r = split_launch(ctx, dp, s, cs, walk, state, train, cnt, tot)) return r;
        final_walk.assign(n, 0);
        launch_lo = {0, cnt.pkgs};
        map_off = {0};
        seg_of.resize(n);
        for (size_t k = 0; k < n; ++k) seg_of[k] = (uint32_t)k;
        rewalks = rounds = 0;
        // rounds: every stream's first segment whose seed was rejected is walked again from its predecessor's end state
        std::vector<uint8_t> eq(n, 1);
        if (!cnt.overflow)
            if (int r = split_compare(ctx, later, eq)) return r;
        auto frontier = [&](size_t k, std::vector<uint32_t> &out) { // the first rejected segment from k on, in k's stream
            for (; k < n && p.first[k] == p.first[k - 1]; ++k)
                if (!eq[k]) {
                    out.push_back((uint32_t)k);
                    return;
                }
        };
        std::vector<uint32_t> rw, next, succ;
        for (size_t k = 0; k < n; ++k)
            if (p.first[k] == k && k + 1 < n) frontier(k + 1, rw);
        while (!rw.empty() && !cnt.overflow) {
            unsigned const m = (unsigned)rw.size(), grid = (m + kSplitWarps - 1) / kSplitWarps;
            rounds++;
            rewalks += m;
            CU(cudaMemcpyAsync(list, rw.data(), m * sizeof(unsigned), cudaMemcpyHostToDevice, st));
            R4_LAUNCH(k_split_gather, grid, kSplitWarps * 32, 0, st, (StreamState const *)state, (int const *)train,
                      (unsigned const *)list, m, rw_state, rw_train, start_seq);
            CU(cudaGetLastError());
            SplitLaunch again; // rw ascends, so its classes stay consecutive
            for (uint32_t k : rw) again.add(walk.off[k], walk.len[k], walk.base[k], true, walk.last[k] != 0, walk.cls[k]);
            if (int r = split_launch(ctx, dp, s, cs, again, rw_state, rw_train, cnt, tot)) return r;
            R4_LAUNCH(k_split_scatter, grid, kSplitWarps * 32, 0, st, (StreamState const *)rw_state, (int const *)rw_train,
                      (unsigned const *)list, m, state, train);
            CU(cudaGetLastError());
            map_off.push_back((uint32_t)seg_of.size());
            seg_of.insert(seg_of.end(), rw.begin(), rw.end());
            launch_lo.push_back(cnt.pkgs);
            succ.clear();
            for (uint32_t k : rw) {
                final_walk[k] = rounds;
                if (k + 1 < n && p.first[k + 1] == p.first[k]) succ.push_back(k + 1);
            }
            if (int r = split_compare(ctx, succ, eq)) return r;
            next.clear();
            for (uint32_t k : succ) frontier(k, next);
            rw.swap(next);
        }
        if (!cnt.overflow) break;
        // an arena was too small: the counters hold what the launches so far needed, the launches still to come more
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)cnt.pkgs * 2 + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)cnt.pool * 2 + 4096);
        if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "package arena overflow");
    }

    // the merge: the packages of every segment's last walk, renumbered, into a second set of arenas that then swaps in.
    // Segments are in internal order and carry the batch's stream index, so the merged packages are in (internal
    // stream, seq) order: every sample rate's streams are one range.
    size_t const n_launch = launch_lo.size() - 1, n_src = launch_lo.back();
    std::vector<uint32_t> tab;
    tab.reserve(3 * n + 2 * n_launch + 1 + seg_of.size() + 1);
    tab.insert(tab.end(), p.stream.begin(), p.stream.end());
    tab.insert(tab.end(), p.first.begin(), p.first.end());
    tab.insert(tab.end(), final_walk.begin(), final_walk.end());
    tab.insert(tab.end(), launch_lo.begin(), launch_lo.end());
    tab.insert(tab.end(), map_off.begin(), map_off.end());
    tab.insert(tab.end(), seg_of.begin(), seg_of.end());
    tab.push_back(0); // the pool cursor
    if (int r = dev_reserve(ctx, ctx->d_sp_tab, tab.size() * sizeof(uint32_t))) return r;
    if (int r = dev_reserve(ctx, ctx->d_sp_pkgs, ctx->pkg_cap * sizeof(r433b_package))) return r;
    if (int r = dev_reserve(ctx, ctx->d_sp_ppool, ctx->pool_cap * sizeof(int))) return r;
    if (int r = dev_reserve(ctx, ctx->d_sp_gpool, ctx->pool_cap * sizeof(int))) return r;
    CU(cudaMemcpyAsync(ctx->d_sp_tab.p, tab.data(), tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    unsigned const *t = (unsigned const *)ctx->d_sp_tab.p;
    SplitMerge mg{};
    mg.n_segs = (unsigned)n;
    mg.n_launches = (unsigned)n_launch;
    mg.seg_stream = t;
    mg.seg_first = t + n;
    mg.final_walk = t + 2 * n;
    mg.launch_lo = t + 3 * n;
    mg.map_off = mg.launch_lo + n_launch + 1;
    mg.seg_of = mg.map_off + n_launch;
    mg.pool_cursor = (unsigned *)ctx->d_sp_tab.p + tab.size() - 1;
    mg.start_seq = start_seq;
    mg.state = state;
    mg.pkg_base = pkg_base;
    mg.src = (r433b_package const *)ctx->d_pkgs.p;
    mg.src_pulse = (int const *)ctx->d_ppool.p;
    mg.src_gap = (int const *)ctx->d_gpool.p;
    mg.dst = (r433b_package *)ctx->d_sp_pkgs.p;
    mg.dst_pulse = (int *)ctx->d_sp_ppool.p;
    mg.dst_gap = (int *)ctx->d_sp_gpool.p;
    CU(cudaEventRecord(ctx->ev_t[3], st));
    R4_LAUNCH(k_split_merge_scan, 1, 32, 0, st, mg);
    if (n_src) R4_LAUNCH(k_split_merge, (unsigned)((n_src + kSplitWarps - 1) / kSplitWarps), kSplitWarps * 32, 0, st, mg);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev_t[4], st));
    std::vector<unsigned> merged(n + 1); // pkg_base: where each segment's packages start, + the total
    unsigned pool_kept = 0;
    CU(cudaMemcpyAsync(merged.data(), pkg_base, (n + 1) * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&pool_kept, mg.pool_cursor, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::swap(ctx->d_pkgs, ctx->d_sp_pkgs);
    std::swap(ctx->d_ppool, ctx->d_sp_ppool);
    std::swap(ctx->d_gpool, ctx->d_sp_gpool);
    if (int r = check_pair_index(ctx, merged[n])) return r;
    ctx->n_pkgs = merged[n];
    ctx->pool_used = pool_kept;
    std::vector<GroupRange> ranges(cs.rate_first.size() - 1);
    for (size_t g = 0; g < ranges.size(); ++g) {
        ranges[g].pkg_begin = merged[stream_seg[cs.rate_first[g]]];
        ranges[g].pkg_end = merged[stream_seg[cs.rate_first[g + 1]]];
    }
    if (int r = slice_ranges(ctx, ranges, ctx->n_pkgs, ctx->pool_used, st)) return r;
    if (ch) {
        R4_LAUNCH(k_split_chain_out, (unsigned)((ns + kSplitWarps - 1) / kSplitWarps), kSplitWarps * 32, 0, st,
                  (StreamState const *)state, (int const *)train, (unsigned const *)slot_first, (unsigned const *)slot_last,
                  (unsigned const *)start_seq, (unsigned const *)pkg_base, (unsigned)ns, (StreamState *)ch->d_state.p,
                  (int *)ch->d_train.p);
        CU(cudaGetLastError());
    }

    // the pass-0 shortcuts count too
    cnt.front_redone += warm_cnt.front_redone;
    cnt.front_repairs += warm_cnt.front_repairs;
    cnt.idle_skipped += warm_cnt.idle_skipped;
    cnt.idle_rewalks += warm_cnt.idle_rewalks;
    cnt.chain_folds += warm_cnt.chain_folds;
    cnt.chain_fm_rebuilds += warm_cnt.chain_fm_rebuilds;
    cudaEventElapsedTime(&ctx->timing.h2d_ms, ctx->ev[0], ctx->ev[1]);
    cudaEventElapsedTime(&ctx->timing.split_merge_ms, ctx->ev_t[3], ctx->ev_t[4]);
    cudaEventElapsedTime(&ctx->timing.total_ms, ctx->ev[0], ctx->ev[3]);
    ctx->timing.front_ms = tot.front_ms;
    ctx->timing.detect_ms = tot.detect_ms;
    ctx->timing.detect_launches = tot.launches;
    ctx->timing.split_segments = (uint32_t)n;
    ctx->timing.split_rewalks = rewalks;
    ctx->timing.split_rounds = rounds;
    return R433B_OK;
}

// rtl_433 -r on every stream of the batch; with a chain, stream i is the next chunk of slot i's file (r433b.h)
int process_iq(r433b_ctx *ctx, r433b_batch const *b, r433b_chain *ch, uint8_t const *last)
{
    Shape s{};
    if (int r = check_batch(ctx, b, ch, last, s)) return r;
    CU(cudaSetDevice(ctx->device));
    if (int r = adopt_batch(ctx, b, s)) return r;
    DetectParams dp{};
    if (int r = prepare_detect(ctx, b, s, dp)) return r;
    if (int r = chain_begin(ctx, ch, last, dp)) return r;
    // slicer parameters: per device, scaled to this batch's sample rate on the host
    if (int r = upload_slicer_tables(ctx, std::vector<uint32_t>{b->samp_rate}, 0)) return r;
    ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, ctx->min_caps[0] ? ctx->min_caps[0] : (size_t)b->n_streams * 16 + 1024);
    ctx->pool_cap = std::max<size_t>(ctx->pool_cap, ctx->min_caps[1] ? ctx->min_caps[1] : ctx->pkg_cap * 128);
    ctx->arena_cap = std::max<size_t>(ctx->arena_cap, ctx->min_caps[2] ? ctx->min_caps[2] : s.total_bytes / 2 + (1u << 20));
    ctx->timing.split_segments = ctx->timing.split_rewalks = ctx->timing.split_rounds = 0;
    ctx->timing.split_merge_ms = 0;
    ctx->timing.mixed_classes = 0;
    ctx->timing.mixed_order_ms = 0;
    DetectCounters cnt{};
    int r = kFellBack;
    SplitPlan plan;
    // a chain splits only when it opted in (r433b_chain_split): the context's setting is for unchained batches
    uint32_t const split_blocks = ch ? ch->split_blocks : ctx->split_blocks, split_warmup = ch ? ch->split_warmup : ctx->split_warmup;
    if (plan_split(ctx, b, s, split_blocks, split_warmup, plan)) {
        ClassSet const cs{{MixedClass{b->samp_rate, (uint32_t)s.SS, (uint32_t)dp.flip, s.fmt.fpdm, 0, 0, b->n_streams, s.max_samples}},
                          {dp.data, dp.data}, {0, b->n_streams}};
        CU(cudaEventRecord(ctx->ev[0], 0));
        r = copy_in(ctx, b, s, 0);
        CU(cudaEventRecord(ctx->ev[1], 0));
        if (!r) r = run_split(ctx, b, s, plan, cs, dp, ch, last, cnt);
    } else {
        uint64_t slice_samples;
        int const G = time_slices(ctx, b, s, slice_samples);
        if (G > 1) r = run_time_sliced(ctx, b, s, G, slice_samples, dp, cnt);
        if (r == kFellBack) r = run_sequential(ctx, b, s, dp, ch, G > 1, cnt);
    }
    if (r) return r;
    ctx->timing.front_redone = cnt.front_redone;
    ctx->timing.front_repairs = cnt.front_repairs;
    ctx->timing.idle_skipped = cnt.idle_skipped;
    ctx->timing.idle_rewalks = cnt.idle_rewalks;
    ctx->timing.chain_folds = cnt.chain_folds;
    ctx->timing.chain_fm_rebuilds = cnt.chain_fm_rebuilds;
    ctx->timing.front_launches = ctx->timing.detect_launches;
    ctx->timing.d2h_ms = 0; // r433b_fetch()'s, or overlapped
    ctx->n_samples = s.used_bytes / s.SS;
    ctx->processed = true;
    return chain_finish(ctx, ch, last, s.settings, std::vector<SlotFormat>(b->n_streams, s.fmt), false);
}

// ---- mixed batches (r433b_process_mixed, DESIGN §7d) -----------------------------------------------------------------

// What the setup of a mixed batch leaves to its schedule (the unsplit class launches, or the split schedule)
struct MixedBatch {
    ChainSettings settings;
    std::vector<SlotFormat> slots;   // per caller stream
    std::vector<uint32_t> order;     // the caller's index of internal stream j
    ClassSet cs;
    std::vector<uint32_t> rates;     // distinct rates ascending; rate slot g starts at internal stream cs.rate_first[g]
    std::vector<uint64_t> conv;      // per caller stream: where its cs16 bytes lie in the conversion region, or UINT64_MAX
    uint64_t conv_base = 0, n_samples = 0;
    uint32_t n_classes = 0;          // distinct (rate, SS, flip, fpdm): launches over both buffers count once
    unsigned *start_seq = nullptr, *internal_of = nullptr;
    unsigned char *slot_cont = nullptr;
    DetectParams dp{};
};

// A mixed batch's arguments, the context's record of the batch, its internal order and classes, the device tables in
// that order, the slicer tables per rate and the detector's parameters.  With a chain, stream i is the next chunk of
// slot i's file: chain_begin() permutes its flags and bases.
int mixed_setup(r433b_ctx *ctx, r433b_batch const *b, r433b_stream_format const *fmt, r433b_chain *ch,
        uint8_t const *last, MixedBatch &m)
{
    if (!ctx || !b || !b->offsets || (b->n_streams && (!b->data || !fmt))) return fail(ctx, R433B_EINVAL, "null argument");
    if (b->sample_format || b->samp_rate || b->center_frequency)
        return fail(ctx, R433B_EINVAL, "r433b_process_mixed: the batch's sample_format, samp_rate and center_frequency "
                                       "must be 0 (each stream has its own)");
    if (b->want_stages) return fail(ctx, R433B_EINVAL, "r433b_process_mixed: no stage arrays (want_stages)");
    uint32_t const n = b->n_streams;
    uint32_t const block_bytes = b->block_bytes ? b->block_bytes : 262144u;
    uint64_t const total = n ? b->offsets[n] : 0;
    if (total % 16) return fail(ctx, R433B_EINVAL, "offsets[n_streams] must be a multiple of 16 bytes");
    int enable_fm = 0;
    for (auto const &d : ctx->devs)
        if (d.modulation >= 16) enable_fm = 1;
    // per stream: checks, its class key, its bytes after conversion (cf32 -> cs16, in the conversion region)
    std::vector<MixedClass> key(n);
    std::vector<uint64_t> len(n), in_lens(n);
    m.conv.assign(n, UINT64_MAX);
    uint64_t conv_bytes = 0;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t const f = fmt[i].sample_format;
        if (f != R433B_FMT_CU8 && f != R433B_FMT_CS16 && f != R433B_FMT_CS8 && f != R433B_FMT_CF32)
            return fail(ctx, R433B_EINVAL, "sample_format must be R433B_FMT_CU8, _CS8, _CS16 or _CF32");
        if (fmt[i].samp_rate == 0) return fail(ctx, R433B_EINVAL, "samp_rate is 0");
        uint32_t const SS = f & 0xff, in_div = f == R433B_FMT_CF32 ? 2 : 1;
        if (block_bytes % (uint32_t)(kTile * SS) != 0)
            return fail(ctx, R433B_EINVAL, "block_bytes must be a multiple of 2048 samples of every sample size in the batch");
        if (b->offsets[i] % (16 * in_div)) return fail(ctx, R433B_EINVAL, "stream offsets must be multiples of 16 bytes (32 for cf32)");
        uint64_t const in_len = b->lengths ? b->lengths[i] : b->offsets[i + 1] - b->offsets[i];
        if (!b->lengths && b->offsets[i + 1] < b->offsets[i]) return fail(ctx, R433B_EINVAL, "offsets not ascending");
        if (b->offsets[i] > total || in_len > total - b->offsets[i])
            return fail(ctx, R433B_EINVAL, "a stream ends behind offsets[n_streams]");
        in_lens[i] = in_len;
        len[i] = in_div == 2 ? in_len / 8 * 4 : in_len; // whole IQ pairs of floats -> cs16 bytes
        if (in_div == 2) {
            m.conv[i] = conv_bytes;
            conv_bytes += (len[i] + 15) / 16 * 16;
        }
        uint32_t const fpdm = b->fpdm_mode == R433B_FPDM_AUTO ? (fmt[i].center_frequency > 800000000u ? 1u : 0u) : b->fpdm_mode;
        key[i] = MixedClass{fmt[i].samp_rate, SS, dp_flip_of(f), fpdm, in_div == 2 && b->data_on_device ? 1u : 0u, 0, 0, 0};
    }
    m.settings = ChainSettings{block_bytes, ctx->use_mag, enable_fm, ctx->level_limit, ctx->min_level, ctx->min_snr,
                               ctx->fm_low_pass};
    m.slots.resize(n);
    for (uint32_t i = 0; i < n; ++i) m.slots[i] = SlotFormat{fmt[i].sample_format, fmt[i].samp_rate, fmt[i].center_frequency, key[i].fpdm};
    if (ch)
        if (int r = check_chain(ctx, b, ch, last, m.settings, true, m.slots, in_lens)) return r;
    CU(cudaSetDevice(ctx->device));

    // the batch becomes the context's last one
    ctx->processed = ctx->fetched = false;
    ctx->chained = ctx->pulse_mode = false;
    ctx->chain_last = nullptr;
    ctx->batch = *b;
    ctx->batch.block_bytes = block_bytes;
    ctx->grabs.clear();
    ctx->grab_planned = false;
    ctx->grab_src = nullptr;
    ctx->grab_flip = 0;
    ctx->timing = r433b_timing{};
    ctx->d2h_done = false;
    // device buffers: host input is copied whole to d_data; the converted cf32 streams follow it there (host input) or
    // fill it (device input)
    m.conv_base = b->data_on_device ? 0 : (total + 255) / 256 * 256;
    if (!b->data_on_device || conv_bytes)
        if (int r = dev_reserve(ctx, ctx->d_data, m.conv_base + conv_bytes + 64)) return r;
    uint8_t const *const caller = b->data_on_device ? (uint8_t const *)b->data : (uint8_t const *)ctx->d_data.p;
    uint8_t const *const region = (uint8_t const *)ctx->d_data.p;
    m.cs.bufs[0] = caller;
    m.cs.bufs[1] = region;
    ctx->offsets.assign(n + 1, total);
    ctx->lengths = len;
    ctx->mixed.resize(n);
    uint64_t used = 0;
    for (uint32_t i = 0; i < n; ++i) {
        bool const cv = m.conv[i] != UINT64_MAX;
        ctx->offsets[i] = cv ? m.conv_base + m.conv[i] : b->offsets[i];
        ctx->mixed[i] = r433b_ctx::MixedStream{key[i].SS, fmt[i].samp_rate, fmt[i].center_frequency, key[i].flip,
                                               cv ? region : caller};
        used += len[i];
        m.n_samples += len[i] / key[i].SS;
    }
    ctx->batch.offsets = ctx->offsets.data();
    ctx->batch.lengths = ctx->lengths.data();

    // the internal order and the classes; the device reads the offsets, lengths and AM offsets in that order
    std::vector<uint32_t> &order = m.order;
    order.resize(n);
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    auto less = [&](MixedClass const &x, MixedClass const &y) {
        return std::tie(x.rate, x.SS, x.flip, x.fpdm, x.buf) < std::tie(y.rate, y.SS, y.flip, y.fpdm, y.buf);
    };
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return less(key[x], key[y]); });
    std::vector<MixedClass> &classes = m.cs.classes;
    std::vector<uint32_t> &slot_first = m.cs.rate_first;
    std::vector<uint64_t> view(3 * n + 2);   // offsets (n + 1), lengths, AM offsets (n + 1)
    uint64_t *off = view.data(), *lens = off + n + 1, *amoff = lens + n;
    amoff[0] = 0;
    for (uint32_t j = 0; j < n; ++j) {
        uint32_t const i = order[j];
        if (classes.empty() || !classes.back().same(key[i])) {
            classes.push_back(key[i]);
            classes.back().begin = j;
        }
        if (m.rates.empty() || m.rates.back() != key[i].rate) {
            m.rates.push_back(key[i].rate);
            slot_first.push_back(j);
        }
        classes.back().end = j + 1;
        classes.back().max_samples = std::max<uint64_t>(classes.back().max_samples, len[i] / key[i].SS);
        off[j] = ctx->offsets[i];
        lens[j] = len[i];
        amoff[j + 1] = amoff[j] + (len[i] / key[i].SS + kTile - 1) / kTile * kTile;
    }
    off[n] = 0;
    slot_first.push_back(n);
    for (size_t c = 0; c < classes.size(); ++c)
        m.n_classes += c == 0 || !(classes[c].rate == classes[c - 1].rate && classes[c].SS == classes[c - 1].SS
                                   && classes[c].flip == classes[c - 1].flip && classes[c].fpdm == classes[c - 1].fpdm);
    uint64_t const am_samples = amoff[n];
    size_t const nn = std::max<size_t>(1, n);
    if (int r = dev_reserve(ctx, ctx->d_offsets, (n + 1) * sizeof(uint64_t))) return r;
    if (int r = dev_reserve(ctx, ctx->d_lengths, nn * sizeof(uint64_t))) return r;
    if (int r = dev_reserve(ctx, ctx->d_amoff, (n + 1) * sizeof(uint64_t))) return r;
    if (int r = dev_reserve(ctx, ctx->d_train, nn * kTrainInts * sizeof(int))) return r;
    if (int r = dev_reserve(ctx, ctx->d_log, nn * kLogCap * 2 * sizeof(unsigned))) return r;
    if (int r = dev_reserve(ctx, ctx->d_counters, 64)) return r;
    if (int r = dev_reserve(ctx, ctx->d_am, am_samples * sizeof(int16_t) + 16)) return r;
    if (int r = dev_reserve(ctx, ctx->d_chunks, am_samples / kChunk * sizeof(ChunkInfo) + 16)) return r;
    if (int r = dev_reserve(ctx, ctx->d_tiles, am_samples / kTile * sizeof(TileInfo) + 16)) return r;
    // d_mx_tab: the caller's index of every internal stream, k_mixed_order's bases (n + 1); chained: per internal stream
    // the seq it starts from, per slot its internal stream and whether it continues a file (bytes)
    if (int r = dev_reserve(ctx, ctx->d_mx_tab, (4 * n + 1) * sizeof(uint32_t) + n)) return r;
    CU(cudaMemcpy(ctx->d_offsets.p, off, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (n) CU(cudaMemcpy(ctx->d_lengths.p, lens, n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_amoff.p, amoff, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (n) CU(cudaMemcpy(ctx->d_mx_tab.p, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    m.start_seq = (unsigned *)ctx->d_mx_tab.p + 2 * n + 1;
    m.internal_of = m.start_seq + n;
    m.slot_cont = (unsigned char *)(m.internal_of + n);
    if (ch && n) {
        std::vector<uint32_t> in_of(n);
        for (uint32_t j = 0; j < n; ++j) in_of[order[j]] = j;
        CU(cudaMemcpy(m.internal_of, in_of.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(m.slot_cont, ch->open.data(), n, cudaMemcpyHostToDevice));
    }
    if (int r = upload_slicer_tables(ctx, m.rates, 0)) return r;
    ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, ctx->min_caps[0] ? ctx->min_caps[0] : (size_t)n * 16 + 1024);
    ctx->pool_cap = std::max<size_t>(ctx->pool_cap, ctx->min_caps[1] ? ctx->min_caps[1] : ctx->pkg_cap * 128);
    ctx->arena_cap = std::max<size_t>(ctx->arena_cap, ctx->min_caps[2] ? ctx->min_caps[2] : used / 2 + (1u << 20));

    DetectParams &dp = m.dp;
    dp.offsets = (unsigned long long const *)ctx->d_offsets.p;
    dp.lengths = (unsigned long long const *)ctx->d_lengths.p;
    dp.am_offsets = (unsigned long long const *)ctx->d_amoff.p;
    dp.n_streams = n;
    dp.sample_end = ~0ull;
    dp.first_chunk = 1;
    dp.use_mag = ctx->use_mag;
    dp.enable_fm = enable_fm;
    dp.lv = ctx->lv;
    dp.lpf_a1 = ((int)(0.85408 * 32768)) >> 1; // src/baseband.c:151-152
    dp.lpf_b0 = ((int)(0.07296 * 32768)) >> 1;
    dp.train_scratch = (int *)ctx->d_train.p;
    dp.log_scratch = (unsigned *)ctx->d_log.p;
    dp.counters = (DetectCounters *)ctx->d_counters.p;
    dp.am = (int16_t *)ctx->d_am.p;
    dp.chunks = (ChunkInfo const *)ctx->d_chunks.p;
    dp.tile_info = (TileInfo const *)ctx->d_tiles.p;
    return chain_begin(ctx, ch, last, dp, &order);
}

// The batch to the device on stream 0 between ev[0] and ev[1]: host input in one copy, every cf32 stream converted into
// the region.  A rerun after an arena overflow starts behind it.
int mixed_copy_in(r433b_ctx *ctx, r433b_batch const *b, MixedBatch const &m)
{
    cudaStream_t const st = 0;
    CU(cudaEventRecord(ctx->ev[0], st));
    Shape whole{};
    whole.total_bytes = b->n_streams ? b->offsets[b->n_streams] : 0;
    if (int r = copy_in(ctx, b, whole, st)) return r; // host input: one copy; device input: nothing
    for (uint32_t i = 0; i < b->n_streams; ++i) {
        size_t const n4 = (size_t)(ctx->lengths[i] / 4 + 1) / 2; // two cs16 samples per group of four floats
        if (m.conv[i] == UINT64_MAX || !n4) continue;
        unsigned const grid = (unsigned)std::min<size_t>((size_t)ctx->n_sms * 8, (n4 + 255) / 256);
        R4_LAUNCH(k_cf32_to_cs16, grid, 256, 0, st, (float4 const *)(m.cs.bufs[0] + b->offsets[i]),
                  (uint2 *)((uint8_t *)ctx->d_data.p + m.conv_base + m.conv[i]), n4);
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(ctx->ev[1], st));
    return R433B_OK;
}

// The unsplit schedule of a mixed batch: one k_front + k_detect launch per class (again with the arenas grown to what
// the device counted while they overflow), k_mixed_order, then the slicers over one package range per rate.  A chain's
// slots are gathered into internal order in front of every attempt and scattered back once the batch has succeeded.
int run_mixed(r433b_ctx *ctx, r433b_batch const *b, MixedBatch &m, r433b_chain *ch, DetectCounters &cnt)
{
    cudaStream_t const st = 0;
    uint32_t const n = b->n_streams;
    DetectParams &dp = m.dp;
    for (int attempt = 0;; ++attempt) {
        if (int r = bind_detector_arenas(ctx, dp)) return r;
        CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, st));
        if (ch) { // from the chain, which only the scatter below writes: also where an overflow reruns from
            CU(cudaMemsetAsync(m.start_seq, 0, n * sizeof(unsigned), st));
            R4_LAUNCH(k_split_chain_in, (n + kSplitWarps - 1) / kSplitWarps, kSplitWarps * 32, 0, st,
                      (StreamState const *)ch->d_state.p, (int const *)ch->d_train.p, (unsigned char const *)m.slot_cont,
                      (unsigned const *)m.internal_of, n, (StreamState *)dp.state, dp.train_scratch, m.start_seq);
            CU(cudaGetLastError());
        }
        if (int r = launch_classes(ctx, dp, m.cs.classes, m.cs.bufs, m.settings.block_bytes)) return r;
        CU(cudaMemcpyAsync(&cnt, ctx->d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (!cnt.overflow) break;
        // arenas were too small: the counters hold the true need
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)cnt.pkgs + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)cnt.pool + 4096);
        if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "package arena overflow");
    }
    if (int r = check_pair_index(ctx, cnt.pkgs)) return r;
    ctx->n_pkgs = cnt.pkgs;
    ctx->pool_used = cnt.pool;

    // k_mixed_order: the headers by rate slot, with the caller's stream indices
    std::vector<uint32_t> base(n + 1, 0);
    if (int r = dev_reserve(ctx, ctx->d_mx_pkgs, ctx->pkg_cap * sizeof(r433b_package))) return r;
    CU(cudaEventRecord(ctx->ev_t[0], st));
    if (ctx->n_pkgs) {
        MixedOrder mo{};
        mo.src = (r433b_package const *)ctx->d_pkgs.p;
        mo.dst = (r433b_package *)ctx->d_mx_pkgs.p;
        mo.n_pkgs = ctx->n_pkgs;
        mo.n_streams = n;
        mo.caller = (unsigned const *)ctx->d_mx_tab.p;
        mo.base = (unsigned *)ctx->d_mx_tab.p + n;
        mo.start_seq = ch ? m.start_seq : nullptr;
        unsigned const grid = (unsigned)std::min<uint64_t>((uint64_t)ctx->n_sms * 4, (ctx->n_pkgs + kMixedThreads - 1) / kMixedThreads);
        CU(cudaMemsetAsync(mo.base, 0, (n + 1) * sizeof(unsigned), st));
        R4_LAUNCH(k_mixed_order, grid, kMixedThreads, 0, st, mo, 0);
        R4_LAUNCH(k_mixed_order, 1, 32, 0, st, mo, 1);
        R4_LAUNCH(k_mixed_order, grid, kMixedThreads, 0, st, mo, 2);
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(base.data(), mo.base, (n + 1) * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaEventRecord(ctx->ev_t[1], st));
    CU(cudaEventSynchronize(ctx->ev_t[1]));
    std::swap(ctx->d_pkgs, ctx->d_mx_pkgs);
    std::vector<GroupRange> ranges(m.rates.size());
    for (size_t g = 0; g < m.rates.size(); ++g) {
        ranges[g].pkg_begin = base[m.cs.rate_first[g]];
        ranges[g].pkg_end = base[m.cs.rate_first[g + 1]];
    }
    if (int r = slice_ranges(ctx, ranges, ctx->n_pkgs, ctx->pool_used, st)) return r;
    if (ch && n) { // the batch has succeeded: the walks' end states back to their slots
        R4_LAUNCH(k_split_scatter, (n + kSplitWarps - 1) / kSplitWarps, kSplitWarps * 32, 0, st,
                  (StreamState const *)dp.state, (int const *)dp.train_scratch, (unsigned const *)ctx->d_mx_tab.p, n,
                  (StreamState *)ch->d_state.p, (int *)ch->d_train.p);
        CU(cudaGetLastError());
    }

    class_spans(ctx, m.cs.classes.size(), ctx->timing.front_ms, ctx->timing.detect_ms);
    ctx->timing.h2d_ms = elapsed_ms(ctx->ev[0], ctx->ev[1]);
    ctx->timing.total_ms = elapsed_ms(ctx->ev[0], ctx->ev[3]);
    ctx->timing.mixed_order_ms = elapsed_ms(ctx->ev_t[0], ctx->ev_t[1]);
    ctx->timing.detect_launches = (uint32_t)m.cs.classes.size();
    return R433B_OK;
}

// rtl_433 -r f1 -r f2 ... on a batch of files of their own formats (DESIGN §7d).  Unchained, with splitting on
// (r433b_set_split) and a stream of two segments, the split schedule walks the segments of every class in the same
// passes; otherwise every class is one launch.  With a chain, stream i is the next chunk of slot i's file; a chain
// runs unsplit.
int process_mixed(r433b_ctx *ctx, r433b_batch const *b, r433b_stream_format const *fmt, r433b_chain *ch,
        uint8_t const *last)
{
    MixedBatch m;
    if (int r = mixed_setup(ctx, b, fmt, ch, last, m)) return r;
    if (int r = mixed_copy_in(ctx, b, m)) return r;
    DetectCounters cnt{};
    Shape s{};
    s.settings = m.settings;
    SplitPlan plan;
    if (!ch && plan_split(ctx, b, s, ctx->split_blocks, ctx->split_warmup, plan, &m.order)) {
        if (int r = run_split(ctx, b, s, plan, m.cs, m.dp, nullptr, nullptr, cnt)) return r;
    } else if (int r = run_mixed(ctx, b, m, ch, cnt)) {
        return r;
    }
    ctx->timing.mixed_classes = m.n_classes;
    ctx->timing.front_launches = ctx->timing.detect_launches;
    ctx->timing.front_redone = cnt.front_redone;
    ctx->timing.front_repairs = cnt.front_repairs;
    ctx->timing.idle_skipped = cnt.idle_skipped;
    ctx->timing.idle_rewalks = cnt.idle_rewalks;
    ctx->timing.chain_folds = cnt.chain_folds;
    ctx->timing.chain_fm_rebuilds = cnt.chain_fm_rebuilds;
    ctx->n_samples = m.n_samples;
    ctx->processed = true;
    return chain_finish(ctx, ch, last, m.settings, m.slots, true);
}

} // namespace

int r433b_process(r433b_ctx *ctx, r433b_batch const *b) { return process_iq(ctx, b, nullptr, nullptr); }
int r433b_process_mixed(r433b_ctx *ctx, r433b_batch const *b, r433b_stream_format const *fmt)
{
    return process_mixed(ctx, b, fmt, nullptr, nullptr);
}

int r433b_chain_create(r433b_ctx *ctx, uint32_t n_streams, r433b_chain **out)
{
    if (!ctx || !out || !n_streams) return fail(ctx, R433B_EINVAL, "r433b_chain_create: null argument or no streams");
    *out = nullptr;
    CU(cudaSetDevice(ctx->device));
    r433b_chain *ch = new (std::nothrow) r433b_chain();
    if (!ch) return R433B_ENOMEM;
    ch->ctx = ctx;
    ctx->chains.push_back(ch);
    ch->n = n_streams;
    ch->open.assign(n_streams, 0);
    ch->next.assign(n_streams, 0);
    ch->fmt.assign(n_streams, SlotFormat{});
    size_t const n = n_streams;
    for (auto [buf, bytes] : {std::pair<DevBuf *, size_t>{&ch->d_state, n * sizeof(StreamState)}, {&ch->d_state_copy, n * sizeof(StreamState)},
                              {&ch->d_train, n * kTrainInts * sizeof(int)}, {&ch->d_train_copy, n * kTrainInts * sizeof(int)},
                              {&ch->d_flags, 2 * n}, {&ch->d_base, n * sizeof(uint64_t)}})
        if (int r = dev_reserve(ctx, *buf, bytes)) {
            r433b_chain_destroy(ch);
            return r;
        }
    *out = ch;
    return R433B_OK;
}

void r433b_chain_destroy(r433b_chain *ch)
{
    if (!ch) return;
    if (r433b_ctx *ctx = ch->ctx) {
        ctx->chains.erase(std::remove(ctx->chains.begin(), ctx->chains.end(), ch), ctx->chains.end());
        if (ctx->chain_last == ch) ctx->chain_last = nullptr;
        cudaSetDevice(ctx->device);
        chain_free_device(ch);
    }
    delete ch;
}

int r433b_process_chained(r433b_ctx *ctx, r433b_batch const *b, r433b_chain *chain, uint8_t const *last)
{
    if (!chain || !chain->ctx) return fail(ctx, R433B_EINVAL, "r433b_process_chained: no chain, or its context is gone");
    return process_iq(ctx, b, chain, last);
}

int r433b_process_mixed_chained(r433b_ctx *ctx, r433b_batch const *b, r433b_stream_format const *fmt, r433b_chain *chain,
        uint8_t const *last)
{
    if (!chain || !chain->ctx)
        return fail(ctx, R433B_EINVAL, "r433b_process_mixed_chained: no chain, or its context is gone");
    return process_mixed(ctx, b, fmt, chain, last);
}

int r433b_chain_grab(r433b_chain *chain, int mode)
{
    if (!chain || !chain->ctx) return R433B_EINVAL;
    r433b_ctx *ctx = chain->ctx;
    if (mode < R433B_GRAB_ALL || mode > R433B_GRAB_UNDECODED) return fail(ctx, R433B_EINVAL, "grab mode must be 1 .. 4");
    if (chain->grab_mode) return fail(ctx, R433B_ESTATE, "r433b_chain_grab: the chain grabs already, in a fixed mode");
    if (std::find(chain->open.begin(), chain->open.end(), 1) != chain->open.end())
        return fail(ctx, R433B_ESTATE, "r433b_chain_grab while a file of the chain is open");
    CU(cudaSetDevice(ctx->device));
    size_t const n = chain->n;
    try { // host state first: a failure past this point has only device memory to give back

        chain->run.assign(n, 0);
        chain->run_c0.assign(n, 0);
        chain->pre_lo.assign(n, 0);
        chain->pre_off.assign(n, 0);
        chain->frame.assign(n, GrabFrame{});
        chain->frame_next.assign(n, GrabFrame{});
        chain->counter.assign(n, 1); // samp_grab_create()
        chain->counter_next.assign(n, 1);
        chain->ended.assign(n, 0);
    } catch (std::exception const &) {
        return fail(ctx, R433B_ENOMEM, "r433b_chain_grab: out of host memory");
    }
    cudaError_t e = cudaMalloc(&chain->d_ring.p, n * kGrabRingBytes);
    if (e != cudaSuccess) {
        chain->d_ring = DevBuf{};
        return fail(ctx, R433B_ENOMEM, "r433b_chain_grab: cudaMalloc of the rings", e);
    }
    chain->d_ring.cap = n * kGrabRingBytes;
    if (int r = dev_reserve(ctx, chain->d_ring_slots, n * sizeof(GrabRingSlot))) {
        cudaFree(chain->d_ring.p);
        chain->d_ring = DevBuf{};
        return r;
    }
    chain->grab_mode = mode;
    chain->grab_pending = false;
    return R433B_OK;
}

int r433b_chain_base(r433b_chain const *chain, uint32_t stream, uint64_t *first_sample)
{
    if (!chain || !first_sample || stream >= chain->n) return R433B_EINVAL;
    *first_sample = stream < chain->base.size() ? chain->base[stream] : 0;
    return R433B_OK;
}

int r433b_get_counts(r433b_ctx const *ctx, uint64_t out[4])
{
    if (!ctx || !out) return R433B_EINVAL;
    if (!ctx->processed) return R433B_ESTATE;
    out[0] = ctx->n_pkgs;
    out[1] = ctx->n_events;
    out[2] = ctx->event_bytes;
    out[3] = ctx->n_samples;
    return R433B_OK;
}

int r433b_get_timing(r433b_ctx const *ctx, r433b_timing *out)
{
    if (!ctx || !out) return R433B_EINVAL;
    *out = ctx->timing;
    return R433B_OK;
}

int r433b_fetch(r433b_ctx *ctx, r433b_results *out)
{
    if (!ctx || !out) return R433B_EINVAL;
    if (!ctx->processed) return fail(ctx, R433B_ESTATE, "r433b_fetch before r433b_process");
    CU(cudaSetDevice(ctx->device));
    cudaStream_t const st = 0;
    uint32_t const n_devs = (uint32_t)ctx->devs.size();
    GroupRange all{};
    all.pkg_end = ctx->n_pkgs;
    all.pool_end = ctx->pool_used;
    all.arena_end = ctx->event_bytes;
    CU(cudaEventRecord(ctx->ev[4], st));
    for (ResultPart const &p : result_parts(ctx, all))
        if (int r = host_reserve(ctx, p.h, p.hi + 16)) return r;
    if (!ctx->d2h_done) {
        if (int r = copy_results(ctx, all, st)) return r;
        ctx->d2h_done = true;
    }
    CU(cudaEventRecord(ctx->ev[5], st));
    CU(cudaEventSynchronize(ctx->ev[5]));
    cudaEventElapsedTime(&ctx->timing.d2h_ms, ctx->ev[4], ctx->ev[5]);
    // the device wrote packages in completion order; the reference's order is per stream
    r433b_package *pk = (r433b_package *)ctx->h_pkgs.p;
    if (!ctx->fetched) {
        // sort an index, then permute: dev_index remembers where each package sits on the device (r433b_analyze)
        std::vector<uint32_t> &ix = ctx->dev_index;
        ix.resize(ctx->n_pkgs);
        for (uint32_t i = 0; i < ctx->n_pkgs; ++i) ix[i] = i;
        std::sort(ix.begin(), ix.end(), [pk](uint32_t a, uint32_t b) {
            return pk[a].stream != pk[b].stream ? pk[a].stream < pk[b].stream : pk[a].seq < pk[b].seq;
        });
        std::vector<r433b_package> sorted(ctx->n_pkgs);
        for (uint32_t i = 0; i < ctx->n_pkgs; ++i) sorted[i] = pk[ix[i]];
        if (ctx->n_pkgs) memcpy(pk, sorted.data(), (size_t)ctx->n_pkgs * sizeof(r433b_package));
        ctx->analyzed = false;
        ctx->p_events.assign(ctx->n_pkgs, 0);
        ctx->dispatched.assign(ctx->batch.n_streams, 0);
    }
    ctx->fetched = true;
    out->n_packages = ctx->n_pkgs;
    out->n_devices = n_devs;
    out->packages = pk;
    out->pulse_pool = (int32_t const *)ctx->h_ppool.p;
    out->gap_pool = (int32_t const *)ctx->h_gpool.p;
    out->pairs = (r433b_pair const *)ctx->h_pairs.p;
    out->events = (uint8_t const *)ctx->h_events.p;
    out->event_bytes = ctx->event_bytes;
    out->n_events = ctx->n_events;
    out->n_samples = ctx->n_samples;
    out->n_gated = ctx->n_gated;
    return R433B_OK;
}

int r433b_copy_stage(r433b_ctx *ctx, uint32_t stream, int16_t *am, int16_t *fm, uint64_t max_samples)
{
    if (!ctx || !am || !fm) return R433B_EINVAL;
    if (!ctx->processed || !ctx->batch.want_stages) return fail(ctx, R433B_ESTATE, "no stage arrays kept (batch.want_stages)");
    if (stream >= ctx->batch.n_streams) return fail(ctx, R433B_EINVAL, "stream out of range");
    CU(cudaSetDevice(ctx->device));
    uint64_t SS = ctx->batch.sample_format;
    uint64_t first = ctx->offsets[stream] / SS;
    uint64_t n = ctx->lengths[stream] / SS;
    if (n > max_samples) n = max_samples;
    if (n) {
        CU(cudaMemcpy(am, (int16_t const *)ctx->d_am.p + ctx->am_offsets[stream], n * sizeof(int16_t), cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(fm, (int16_t const *)ctx->d_fm.p + first, n * sizeof(int16_t), cudaMemcpyDeviceToHost));
    }
    return (int)std::min<uint64_t>(n, 0x7fffffff);
}

// ------------------------------------------------------------------ host-side replay ------

int r433b_event_to_bitbuffer(uint8_t const *ev, uint32_t pair_bytes, uint32_t index, struct bitbuffer *out,
        uint32_t *consumed)
{
    return event_to_bitbuffer(ev, pair_bytes, index, out, consumed);
}

float r433b_package_file_pos(r433b_ctx const *ctx, r433b_results const *res, uint32_t package)
{
    if (!ctx || !res || package >= res->n_packages) return 0.0f;
    if (ctx->pulse_mode) return 0.0f; // demod->sample_file_pos = 0.0 in front of the .ook loop, src/rtl_433.c:1752
    r433b_package const &k = res->packages[package];
    StreamFormat const f = stream_format(ctx, k.stream);
    uint64_t SS = f.SS;
    // a chained chunk: the bytes of its file up to the chunk's end (k.block is absolute)
    uint64_t bytes = ctx->lengths[k.stream] + (ctx->chained ? ctx->chain_base[k.stream] * SS : 0);
    uint32_t bb = ctx->batch.block_bytes;
    uint64_t n_blocks = (bytes + bb - 1) / bb;
    if (n_blocks == 0) return 0.0f;
    // src/rtl_433.c:1839: value set before the block that returned the package was pushed;
    // the flush keeps the last block's value
    uint64_t blk = (uint64_t)k.block < n_blocks ? (uint64_t)k.block : n_blocks - 1;
    unsigned long n_read = (unsigned long)std::min<uint64_t>(bb, bytes - blk * bb);
    float pos = ((float)(int)blk * bb + n_read) / f.rate / (int)SS;
    return pos;
}

int r433b_package_to_pulse_data(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, struct pulse_data *pd)
{
    if (!ctx || !res || !pd || package >= res->n_packages) return R433B_EINVAL;
    r433b_package const &k = res->packages[package];
    memset(pd, 0, sizeof(*pd));
    if (ctx->pulse_mode) {
        // a loaded package: exactly what pulse_data_load() / rfraw_parse() left in the struct
        if (k.end_pos >= ctx->pulse_meta.size()) return R433B_EINVAL;
        PulseSet::Meta const &m = ctx->pulse_meta[k.end_pos];
        pd->sample_rate = m.rate;
        pd->num_pulses = m.num_pulses;
        memcpy(pd->pulse, res->pulse_pool + k.pulse_off, k.pulse_count * sizeof(int));
        memcpy(pd->gap, res->gap_pool + k.pulse_off, k.pulse_count * sizeof(int));
        pd->fsk_f1_est = m.fsk_f1_est;
        pd->fsk_f2_est = m.fsk_f2_est;
        pd->freq1_hz = m.freq1_hz;
        pd->freq2_hz = m.freq2_hz;
        return R433B_OK;
    }
    StreamFormat const f = stream_format(ctx, k.stream);
    pd->offset = k.offset;
    pd->sample_rate = f.rate;
    pd->start_ago = k.start_ago;
    pd->end_ago = k.end_ago;
    pd->num_pulses = k.num_pulses;
    memcpy(pd->pulse, res->pulse_pool + k.pulse_off, k.pulse_count * sizeof(int));
    memcpy(pd->gap, res->gap_pool + k.pulse_off, k.pulse_count * sizeof(int));
    pd->ook_low_estimate = k.ook_low_estimate;
    pd->ook_high_estimate = k.ook_high_estimate;
    pd->fsk_f1_est = k.fsk_f1_est;
    pd->fsk_f2_est = k.fsk_f2_est;
    // calc_rssi_snr(), src/r_flow.c:35-64 (float32, log10f)
    float hi = pd->ook_high_estimate > 0 ? pd->ook_high_estimate : 1;
    float lo = pd->ook_low_estimate > 0 ? pd->ook_low_estimate : 1;
    int const max_high = ctx->lv.max_high;
    float top = hi < max_high ? hi : max_high;
    float asnr = top / lo;
    uint32_t rate = f.rate, center = f.center;
    float off1 = (float)pd->fsk_f1_est / INT16_MAX * rate / 2.0f;
    float off2 = (float)pd->fsk_f2_est / INT16_MAX * rate / 2.0f;
    pd->freq1_hz = off1 + center;
    pd->freq2_hz = off2 + center;
    pd->centerfreq_hz = center;
    pd->depth_bits = f.SS * 4;
    if (f.SS == 2 && !ctx->use_mag) {
        pd->range_db = 42.1442f;
        pd->rssi_db = 10.0f * log10f(hi) - 42.1442f;
        pd->noise_db = 10.0f * log10f(lo) - 42.1442f;
        pd->snr_db = 10.0f * log10f(asnr);
    } else {
        pd->range_db = 84.2884f;
        pd->rssi_db = 20.0f * log10f(hi) - 84.2884f;
        pd->noise_db = 20.0f * log10f(lo) - 84.2884f;
        pd->snr_db = 20.0f * log10f(asnr);
    }
    return R433B_OK;
}

} // extern "C"

namespace {

template <class PerEvent, class PerPair>
int replay_stream(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, PerEvent &&per_event, PerPair &&per_pair)
{
    if (!ctx || !res) return R433B_EINVAL;
    if (!ctx->fetched) return fail(ctx, R433B_ESTATE, "dispatch before fetch");
    uint32_t const n_devs = res->n_devices;
    // packages are sorted by (stream, seq)
    r433b_package const *begin = std::lower_bound(res->packages, res->packages + res->n_packages, stream,
            [](r433b_package const &k, uint32_t s) { return k.stream < s; });
    static thread_local struct pulse_data pd;
    static thread_local struct bitbuffer bits;
    for (r433b_package const *k = begin; k != res->packages + res->n_packages && k->stream == stream; ++k) {
        uint32_t pi = (uint32_t)(k - res->packages);
        r433b_package_to_pulse_data(ctx, res, pi, &pd);
        // run_ook_demods()/run_fsk_demods(), src/r_api.c:438-550
        int p_events = 0;
        unsigned next = 0;
        for (unsigned prio = 0; !p_events && prio < 0xffffffffu; prio = next) {
            next = 0xffffffffu;
            for (uint32_t dv = 0; dv < n_devs; ++dv) {
                unsigned dp = ctx->devs[dv].priority;
                if (dp > prio && dp < next) next = dp;
                if (dp != prio) continue;
                if (!device_takes((int)ctx->devs[dv].modulation, k->type)) continue;
                r433b_pair const &pr = res->pairs[(size_t)k->first_pair + dv];
                per_pair(dv, pr); // the slicer of this device ran: its gated events were handed over too (and turned down)
                uint32_t at = 0;
                for (uint32_t e = 0; e < pr.events; ++e) {
                    uint32_t used = 0;
                    int rc = r433b_event_to_bitbuffer(res->events + pr.offset + at, pr.bytes - at, 0, &bits, &used);
                    if (rc) return fail(ctx, rc, "corrupt event stream");
                    at += used;
                    int ret = per_event(pi, dv, &pd, &bits);
                    if (ret < -4) return fail(ctx, R433B_EINVAL, "decoder returned an invalid code (< -4)");
                    if (ret > 0) p_events += ret;
                }
            }
        }
        if (pi < ctx->p_events.size()) ctx->p_events[pi] = (uint32_t)p_events;
    }
    if (stream < ctx->dispatched.size()) ctx->dispatched[stream] = 1;
    return R433B_OK;
}

} // namespace

extern "C" {

// Position-independent checksum of everything the batch holds for one stream: package headers (without the
// fields that say where in the batch they lie), pulse and gap widths, and the events of every
// (package, device) pair in device order, each in the long form of the wire format (event_long_form).  Two streams with the same samples give the same digest wherever
// they sit in a batch.
int r433b_stream_digest(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, uint64_t *digest)
{
    if (!ctx || !res || !digest) return R433B_EINVAL;
    if (!ctx->fetched) return fail(ctx, R433B_ESTATE, "digest before fetch");
    uint64_t h = 1469598103934665603ull; // FNV-1a, 64 bit, over 32-bit words
    auto mix = [&](uint32_t w) {
        h ^= w;
        h *= 1099511628211ull;
    };
    auto mix_words = [&](void const *ptr, size_t n_words) {
        uint32_t const *w = (uint32_t const *)ptr;
        for (size_t i = 0; i < n_words; ++i) mix(w[i]);
    };
    r433b_package const *begin = std::lower_bound(res->packages, res->packages + res->n_packages, stream,
            [](r433b_package const &k, uint32_t s) { return k.stream < s; });
    std::vector<uint32_t> longform;
    for (r433b_package const *k = begin; k != res->packages + res->n_packages && k->stream == stream; ++k) {
        uint32_t const hdr[] = {k->seq, (uint32_t)k->type, (uint32_t)k->block, (uint32_t)k->offset, (uint32_t)(k->offset >> 32),
                                ctx->pulse_mode ? 0u : (uint32_t)k->end_pos, ctx->pulse_mode ? 0u : (uint32_t)(k->end_pos >> 32), k->start_ago, k->end_ago, k->num_pulses,
                                k->pulse_count, (uint32_t)k->ook_low_estimate, (uint32_t)k->ook_high_estimate,
                                (uint32_t)k->fsk_f1_est, (uint32_t)k->fsk_f2_est};
        mix_words(hdr, sizeof(hdr) / 4);
        mix_words(res->pulse_pool + k->pulse_off, k->pulse_count);
        mix_words(res->gap_pool + k->pulse_off, k->pulse_count);
        for (uint32_t dv = 0; dv < res->n_devices; ++dv) {
            r433b_pair const &pr = res->pairs[(size_t)k->first_pair + dv];
            // the events in their long form, so that the digest does not depend on which of them got one-word forms
            longform.clear();
            uint32_t const *ev = reinterpret_cast<uint32_t const *>(res->events + pr.offset);
            for (uint32_t pos = 0, total = pr.bytes / 4; pos < total;) {
                EventHead const e = event_head(ev[pos]);
                if (e.len < 1 || pos + e.len > total || event_long_form(ev + pos, e, longform))
                    return fail(ctx, R433B_EINVAL, "corrupt event stream");
                pos += e.len;
            }
            mix((uint32_t)longform.size() * 4);
            mix(pr.events);
            mix(pr.gated_single);
            mix(pr.gated_multi);
            mix_words(longform.data(), longform.size());
        }
    }
    *digest = h;
    return R433B_OK;
}

int r433b_dispatch(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, r433b_event_fn fn, void *user)
{
    if (!fn) return R433B_EINVAL;
    return replay_stream(ctx, res, stream, [&](uint32_t pk, uint32_t dv, struct pulse_data *pd, struct bitbuffer *bits) {
        return fn(user, pk, dv, pd, bits);
    }, [](uint32_t, r433b_pair const &) {});
}

int r433b_dispatch_r_devices(r433b_ctx *ctx, r433b_results const *res, uint32_t stream, struct r_device *const *devs,
        uint32_t n)
{
    if (!devs || !res || n != res->n_devices) return R433B_EINVAL;
    return replay_stream(ctx, res, stream, [&](uint32_t, uint32_t dv, struct pulse_data *, struct bitbuffer *bits) {
        // account_event(), src/pulse_slicer.c:26-66
        struct r_device *d = devs[dv];
        int ret = 0;
        if (d->decode_fn) ret = d->decode_fn(d, bits);
        d->decode_events += 1;
        if (ret > 0) {
            d->decode_ok += 1;
            d->decode_messages += ret;
        } else if (ret >= -4) {
            d->decode_fails[-ret] += 1;
            ret = 0;
        }
        return ret;
    }, [&](uint32_t dv, r433b_pair const &pr) {
        // gated events: account_event() with the return code the decoder's own length check gives
        if (!(pr.gated_single | pr.gated_multi) || ctx->gates.size() != n) return;
        struct r_device *d = devs[dv];
        r433b_gate const &g = ctx->gates[dv];
        d->decode_events += pr.gated_single + pr.gated_multi;
        d->decode_fails[-g.code_single] += pr.gated_single;
        d->decode_fails[-g.code_multi] += pr.gated_multi;
    });
}

} // extern "C"

// ------------------------------------------------ threaded replay (SURVEY 8(f1)) ------------
extern "C" {

// The replay of different streams is independent: stream s goes to worker s % n_sets, every worker with its OWN decoder
// instances (dev_sets[w][0..n_devs): separately registered r_device structs -- the counters and decoder contexts are
// per instance; the reference's decoders are not re-entrant on one instance).  Within a stream the order is the
// reference's.  The caller sums the per-set statistics.  Returns the first error of any worker.
int r433b_dispatch_r_devices_parallel(r433b_ctx *ctx, r433b_results const *res, struct r_device *const *const *dev_sets,
        uint32_t n_devs, uint32_t n_sets)
{
    if (!ctx || !res || !dev_sets || !n_sets || n_devs != res->n_devices) return R433B_EINVAL;
    if (!ctx->fetched) return fail(ctx, R433B_ESTATE, "dispatch before fetch");
    uint32_t const n_streams = res->n_packages ? res->packages[res->n_packages - 1].stream + 1 : 0;
    std::atomic<int> first_error{0};
    auto work = [&](uint32_t w) {
        for (uint32_t s = w; s < n_streams && !first_error.load(std::memory_order_relaxed); s += n_sets) {
            int rc = r433b_dispatch_r_devices(ctx, res, s, dev_sets[w], n_devs);
            if (rc) {
                int expected = 0;
                first_error.compare_exchange_strong(expected, rc);
            }
        }
    };
    std::vector<std::thread> pool;
    for (uint32_t w = 1; w < n_sets; ++w) pool.emplace_back(work, w);
    work(0);
    for (auto &t : pool) t.join();
    return first_error.load();
}

} // extern "C"

// ------------------------------------------------ pulse-level I/O (SURVEY 8(f4)) -----------
// Packages that never were IQ: `.ook` pulse files and RfRaw lines go straight to the slicers.

extern "C" {

r433b_pulses *r433b_pulses_create(void) { return new (std::nothrow) r433b_pulses(); }

void r433b_pulses_destroy(r433b_pulses *ps) { delete ps; }

void r433b_pulses_clear(r433b_pulses *ps)
{
    if (!ps) return;
    ps->set = PulseSet();
}

int r433b_pulses_load_ook(r433b_pulses *ps, uint32_t stream, char const *text, size_t len, uint32_t samp_rate)
{
    if (!ps || (!text && len) || !samp_rate) return R433B_EINVAL;
    return load_ook_text(ps->set, stream, text, len, samp_rate);
}

int r433b_pulses_load_rfraw(r433b_pulses *ps, uint32_t stream, char const *line)
{
    if (!ps || !line) return R433B_EINVAL;
    if (!rfraw_is(line)) return 0;
    // `pulse_data_t pulse_data = {0}; rfraw_parse(&pulse_data, line);` (src/rtl_433.c:1622-1624, :1639-1641)
    static thread_local struct pulse_data d;
    memset(&d, 0, sizeof(d));
    rfraw_append(&d, line);
    ps->set.add(stream, &d);
    return 1;
}

int r433b_pulses_add(r433b_pulses *ps, uint32_t stream, struct pulse_data const *pd)
{
    if (!ps || !pd) return R433B_EINVAL;
    ps->set.add(stream, pd);
    return 1;
}

uint32_t r433b_pulses_count(r433b_pulses const *ps) { return ps ? (uint32_t)ps->set.pk.size() : 0; }

int r433b_pulses_get(r433b_pulses const *ps, uint32_t index, struct pulse_data *out)
{
    if (!ps || !out || index >= ps->set.pk.size()) return R433B_EINVAL;
    ps->set.get(index, out);
    return R433B_OK;
}

size_t r433b_format_ook(struct pulse_data const *pd, char const *received, char *buf, size_t cap)
{
    return pd ? format_ook(pd, received, buf, cap) : 0;
}

size_t r433b_format_ook_header(char const *created, char *buf, size_t cap) { return format_ook_header(created, buf, cap); }

size_t r433b_format_vcd(struct pulse_data const *pd, int ch_id, char *buf, size_t cap)
{
    return pd ? format_vcd(pd, ch_id, buf, cap) : 0;
}

size_t r433b_format_vcd_header(uint32_t sample_rate, char const *date, char *buf, size_t cap)
{
    return format_vcd_header(sample_rate, date, buf, cap);
}

void r433b_dump_logic_u8(uint8_t *buf, uint64_t len, uint64_t buf_offset, struct pulse_data const *pd, uint8_t bits)
{
    if (buf && pd) dump_logic_u8(buf, len, buf_offset, pd, bits);
}

// run_ook_demods() / run_fsk_demods() on every package of the set (src/rtl_433.c:1755-1790, :1620-1650): the
// slicers of all registered devices on the GPU, results fetched and replayed like those of r433b_process().
// Packages may carry different sample rates (an RfRaw line is 1 MHz whatever the file's rate is): one package
// range per distinct rate, sliced with the device widths scaled to that rate.
int r433b_process_pulses(r433b_ctx *ctx, r433b_pulses const *ps)
{
    if (!ctx || !ps) return fail(ctx, R433B_EINVAL, "null argument");
    CU(cudaSetDevice(ctx->device));
    PulseSet const &set = ps->set;
    uint32_t const n = (uint32_t)set.pk.size();
    uint32_t const n_devs = (uint32_t)ctx->devs.size();
    if (int r = check_pair_index(ctx, n)) return r;
    ctx->processed = ctx->fetched = false;
    ctx->d2h_done = false;
    ctx->pulse_mode = true;
    ctx->grab_planned = false;
    ctx->pulse_meta = set.pk;
    ctx->mixed.clear();
    ctx->batch = r433b_batch{};
    ctx->batch.sample_format = 2;
    ctx->offsets.clear();
    ctx->lengths.clear();
    cudaStream_t const st = 0;

    // device order: by sample rate (stable), so that every rate is one contiguous package range
    std::vector<uint32_t> order(n);
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return set.pk[a].rate < set.pk[b].rate; });
    std::vector<r433b_package> hp(n);
    std::vector<int32_t> pp, gp;
    pp.reserve(set.pulse.size());
    gp.reserve(set.gap.size());
    std::vector<uint32_t> rates;
    std::vector<GroupRange> ranges; // one per rate
    for (uint32_t j = 0; j < n; ++j) {
        PulseSet::Meta const &m = set.pk[order[j]];
        r433b_package &k = hp[j];
        memset(&k, 0, sizeof(k));
        k.stream = m.stream;
        k.seq = m.seq;
        k.type = m.type;
        k.end_pos = order[j];
        k.num_pulses = m.num_pulses;
        k.pulse_off = (uint32_t)pp.size();
        k.pulse_count = m.count;
        k.fsk_f1_est = m.fsk_f1_est;
        k.fsk_f2_est = m.fsk_f2_est;
        k.first_pair = j * n_devs;
        pp.insert(pp.end(), set.pulse.begin() + m.first, set.pulse.begin() + m.first + m.count);
        gp.insert(gp.end(), set.gap.begin() + m.first, set.gap.begin() + m.first + m.count);
        if (rates.empty() || rates.back() != m.rate) {
            rates.push_back(m.rate);
            ranges.push_back(GroupRange{});
            ranges.back().pkg_begin = j;
        }
        ranges.back().pkg_end = j + 1;
    }
    for (uint32_t rate : rates)
        if (!rate) return fail(ctx, R433B_EINVAL, "a package has sample_rate 0");

    ctx->n_pkgs = n;
    ctx->pool_used = (unsigned)pp.size();
    ctx->n_samples = 0;
    ctx->event_bytes = ctx->n_events = ctx->n_gated = 0;
    ctx->timing = r433b_timing{};
    if (n) { // the packages and their widths go to the device even without devices (r433b_analyze needs them)
        if (int r = dev_reserve(ctx, ctx->d_pkgs, (size_t)n * sizeof(r433b_package))) return r;
        if (int r = dev_reserve(ctx, ctx->d_ppool, pp.size() * sizeof(int) + 16)) return r;
        if (int r = dev_reserve(ctx, ctx->d_gpool, gp.size() * sizeof(int) + 16)) return r;
        CU(cudaMemcpyAsync(ctx->d_pkgs.p, hp.data(), (size_t)n * sizeof(r433b_package), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(ctx->d_ppool.p, pp.data(), pp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(ctx->d_gpool.p, gp.data(), gp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        CU(cudaStreamSynchronize(st));
    }
    if (n && n_devs) {
        size_t const arena_min = ctx->min_caps[2] ? ctx->min_caps[2] : (size_t)(1u << 20);
        if (ctx->arena_cap < arena_min) ctx->arena_cap = arena_min;
        if (int r = upload_slicer_tables(ctx, rates, st)) return r;
        if (int r = slice_ranges(ctx, ranges, n, pp.size(), st)) return r;
        ctx->timing.total_ms = ctx->timing.slice_ms;
    }
    ctx->processed = true;
    return R433B_OK;
}

} // extern "C"


// ------------------------------------------------ pulse analyzer (SURVEY 8(f3)) -------------

namespace {

uint32_t package_rate(r433b_ctx const *ctx, r433b_package const &k)
{
    if (ctx->pulse_mode && k.end_pos < ctx->pulse_meta.size()) return ctx->pulse_meta[k.end_pos].rate;
    return stream_format(ctx, k.stream).rate;
}

} // namespace

extern "C" {

int r433b_analyze(r433b_ctx *ctx, r433b_results const *res)
{
    if (!ctx || !res) return R433B_EINVAL;
    if (!ctx->fetched) return fail(ctx, R433B_ESTATE, "r433b_analyze before r433b_fetch");
    CU(cudaSetDevice(ctx->device));
    uint32_t const n = ctx->n_pkgs;
    ctx->an.assign(n, r433b_analysis{});
    ctx->an_guess.assign(n, r433b_guess{});
    ctx->an_text.assign(n, std::string());
    ctx->an_pairs.assign(n, r433b_pair{});
    ctx->an_events.clear();
    ctx->analyzed = true;
    if (!n) return R433B_OK;
    cudaStream_t const st = 0;
    // 1. histograms on the GPU, device package order
    if (int r = dev_reserve(ctx, ctx->d_an, (size_t)n * sizeof(r433b_analysis))) return r;
    AnalyzeParams ap{};
    ap.pkgs = (r433b_package const *)ctx->d_pkgs.p;
    ap.n_pkgs = n;
    ap.pulse_pool = (int const *)ctx->d_ppool.p;
    ap.gap_pool = (int const *)ctx->d_gpool.p;
    ap.out = (r433b_analysis *)ctx->d_an.p;
    unsigned const grid = (unsigned)(((uint64_t)n * 5 + kAnalyzeThreads - 1) / kAnalyzeThreads);
    R4_LAUNCH(k_analyze, grid, kAnalyzeThreads, 0, st, ap);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(ctx->an.data(), ctx->d_an.p, (size_t)n * sizeof(r433b_analysis), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    // 2. the guess and the text on the host (sorted package order -> device order through dev_index)
    std::vector<SlicerParams> sp(n);
    std::vector<int> last_gap(n, -1);
    static thread_local struct pulse_data pd;
    std::vector<char> buf(1 << 16);
    bool any = false;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t const di = ctx->dev_index[i];
        r433b_package_to_pulse_data(ctx, res, i, &pd);
        r433b_guess g{};
        size_t len = analysis_finish(&pd, res->packages[i].type, ctx->an[di], &g, buf.data(), buf.size());
        if (len >= buf.size()) {
            buf.resize(len + 1);
            len = analysis_finish(&pd, res->packages[i].type, ctx->an[di], &g, buf.data(), buf.size());
        }
        ctx->an_text[di].assign(buf.data(), len);
        ctx->an_guess[di] = g;
        sp[di] = SlicerParams{};
        if (g.modulation && g.sliced) {
            r433b_device d{};
            d.modulation = g.modulation;
            d.short_width = g.short_width;
            d.long_width = g.long_width;
            d.reset_limit = g.reset_limit;
            d.gap_limit = g.gap_limit;
            d.sync_width = g.sync_width;
            d.tolerance = g.tolerance;
            sp[di] = scale_device(d, package_rate(ctx, res->packages[i]));
            last_gap[di] = g.last_gap;
            any = true;
        }
    }
    if (!any) return R433B_OK;
    // 3. the trial demodulation: every package through the slicer of its own guess
    if (int r = dev_reserve(ctx, ctx->d_an_dev, (size_t)n * sizeof(SlicerParams))) return r;
    if (int r = dev_reserve(ctx, ctx->d_an_gap, (size_t)n * sizeof(int))) return r;
    if (int r = dev_reserve(ctx, ctx->d_an_pairs, (size_t)n * sizeof(r433b_pair))) return r;
    CU(cudaMemcpyAsync(ctx->d_an_dev.p, sp.data(), (size_t)n * sizeof(SlicerParams), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_an_gap.p, last_gap.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(ctx->d_an_pairs.p, 0, (size_t)n * sizeof(r433b_pair), st));
    OwnSliceParams op{};
    op.pkgs = ap.pkgs;
    op.n_pkgs = n;
    op.pulse_pool = ap.pulse_pool;
    op.gap_pool = (int *)ctx->d_gpool.p;
    op.dev = (SlicerParams const *)ctx->d_an_dev.p;
    op.last_gap = (int const *)ctx->d_an_gap.p;
    op.pairs = (r433b_pair *)ctx->d_an_pairs.p;
    op.arena = nullptr;
    op.pass = 0;
    unsigned const og = (n + 127) / 128;
    R4_LAUNCH(k_slice_own, og, 128, 0, st, op);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(ctx->an_pairs.data(), ctx->d_an_pairs.p, (size_t)n * sizeof(r433b_pair), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    uint64_t total = 0;
    for (auto &pr : ctx->an_pairs) {
        pr.offset = total;
        total += pr.bytes;
    }
    if (total) {
        if (int r = dev_reserve(ctx, ctx->d_an_arena, total)) return r;
        CU(cudaMemcpyAsync(ctx->d_an_pairs.p, ctx->an_pairs.data(), (size_t)n * sizeof(r433b_pair), cudaMemcpyHostToDevice, st));
        op.arena = (uint8_t *)ctx->d_an_arena.p;
        op.pass = 1;
        R4_LAUNCH(k_slice_own, og, 128, 0, st, op);
        CU(cudaGetLastError());
        ctx->an_events.resize(total);
        CU(cudaMemcpyAsync(ctx->an_events.data(), ctx->d_an_arena.p, total, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return R433B_OK;
}

int r433b_analysis_get(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, r433b_analysis *out, r433b_guess *guess)
{
    if (!ctx || !res || !ctx->analyzed || package >= ctx->dev_index.size()) return R433B_EINVAL;
    uint32_t const di = ctx->dev_index[package];
    if (out) *out = ctx->an[di];
    if (guess) *guess = ctx->an_guess[di];
    return R433B_OK;
}

size_t r433b_analysis_text(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, char *buf, size_t cap)
{
    if (!ctx || !res || !ctx->analyzed || package >= ctx->dev_index.size()) return 0;
    std::string const &t = ctx->an_text[ctx->dev_index[package]];
    if (buf && cap) {
        size_t n = t.size() < cap - 1 ? t.size() : cap - 1;
        memcpy(buf, t.data(), n);
        buf[n] = 0;
    }
    return t.size();
}

int r433b_analysis_events(r433b_ctx const *ctx, r433b_results const *res, uint32_t package, uint8_t const **events,
        uint32_t *bytes, uint32_t *n_events)
{
    if (!ctx || !res || !ctx->analyzed || package >= ctx->dev_index.size()) return R433B_EINVAL;
    r433b_pair const &pr = ctx->an_pairs[ctx->dev_index[package]];
    if (events) *events = pr.bytes ? ctx->an_events.data() + pr.offset : nullptr;
    if (bytes) *bytes = pr.bytes;
    if (n_events) *n_events = pr.events;
    return R433B_OK;
}

} // extern "C"


// ------------------------------------------------ asynchronous batches (SURVEY 8(b), 8(f1)) -

extern "C" {

// r433b_process() + r433b_fetch() of `batch` on a worker thread of the context.  The descriptor arrays are copied,
// the sample data is not: it must stay valid until r433b_wait().  One batch in flight per context; until it has
// been waited for, the context must not be touched (the previous batch's results are overwritten while it runs).
// The way to overlap the GPU with the host replay is two contexts on the same device used alternately:
//     submit(A, batch k+1);  dispatch(results of B = batch k);  wait(A);  swap(A, B)
int r433b_submit(r433b_ctx *ctx, r433b_batch const *batch)
{
    if (!ctx || !batch || !batch->offsets) return fail(ctx, R433B_EINVAL, "null argument");
    if (ctx->in_flight) return fail(ctx, R433B_ESTATE, "r433b_submit: a batch is already in flight (r433b_wait first)");
    if (ctx->worker.joinable()) ctx->worker.join();
    ctx->sub_batch = *batch;
    ctx->sub_offsets.assign(batch->offsets, batch->offsets + batch->n_streams + 1);
    ctx->sub_batch.offsets = ctx->sub_offsets.data();
    if (batch->lengths) {
        ctx->sub_lengths.assign(batch->lengths, batch->lengths + batch->n_streams);
        ctx->sub_batch.lengths = ctx->sub_lengths.data();
    }
    ctx->in_flight = true;
    ctx->worker = std::thread([ctx]() {
        int rc = r433b_process(ctx, &ctx->sub_batch);
        if (!rc) rc = r433b_fetch(ctx, &ctx->sub_res);
        ctx->worker_rc = rc;
    });
    return R433B_OK;
}

int r433b_wait(r433b_ctx *ctx, r433b_results *out)
{
    if (!ctx) return R433B_EINVAL;
    if (!ctx->in_flight) return fail(ctx, R433B_ESTATE, "r433b_wait without r433b_submit");
    ctx->worker.join();
    ctx->in_flight = false;
    if (!ctx->worker_rc && out) *out = ctx->sub_res;
    return ctx->worker_rc;
}

} // extern "C"


// ------------------------------------------------ signal grabber (src/samp_grab.c, src/r_flow.c:345-362) ------

namespace {

// The run byte range [a, b) as segments of the staging buffer from `dst` on: negative positions were never written
// (zero), positions before the batch come from the device copy of the prior tail, the rest from the streams' used
// bytes as they lie on the device.  seg_stream gets each segment's stream (UINT32_MAX: not the batch's bytes).
void grab_segments(r433b_ctx const *ctx, int64_t a, int64_t b, uint64_t &dst, std::vector<GrabSeg> &segs,
        std::vector<uint32_t> &seg_stream)
{
    int64_t const pushed = (int64_t)ctx->grab_pushed;
    while (a < b) {
        GrabSeg g{};
        g.dst = dst;
        int64_t e;
        uint32_t stream = UINT32_MAX;
        if (a < 0) {
            e = std::min<int64_t>(b, 0);
            g.kind = kGrabZero;
        } else if (a < pushed) {
            e = std::min<int64_t>(b, pushed);
            g.kind = kGrabPrior;
            g.src = (uint64_t)(a - (pushed - (int64_t)ctx->grab_prior_bytes));
        } else {
            uint64_t const u = (uint64_t)(a - pushed);
            std::vector<uint64_t> const &cum = ctx->grab_cum;
            size_t const s = (size_t)(std::upper_bound(cum.begin(), cum.end(), u) - cum.begin()) - 1;
            e = std::min<int64_t>(b, pushed + (int64_t)cum[s + 1]);
            g.kind = kGrabBatch;
            g.src = ctx->offsets[s] + (u - cum[s]);
            stream = (uint32_t)s;
        }
        g.len = (uint64_t)(e - a);
        seg_stream.push_back(stream);
        segs.push_back(g);
        dst += g.len;
        a = e;
    }
}

// Slot s's run byte range [a, b) on a grabbing chain after its last batch, as segments: negative positions were never
// written (zero); the ring holds the newest kGrabRingBytes (split at its wrap); older bytes of the chunk come from the
// batch, older ones before it from the bytes the append overwrote (saved at d_pre).  seg_stream as in grab_segments.
void chain_grab_segments(r433b_ctx const *ctx, r433b_chain const *ch, uint32_t s, int64_t a, int64_t b, uint64_t &dst,
        std::vector<GrabSeg> &segs, std::vector<uint32_t> &seg_stream)
{
    int64_t const S = kGrabRingBytes, c0 = (int64_t)ch->run_c0[s], ring_lo = (int64_t)ch->run[s] - S;
    while (a < b) {
        GrabSeg g{};
        g.dst = dst;
        int64_t e;
        if (a < 0) {
            e = std::min<int64_t>(b, 0);
            g.kind = kGrabZero;
        } else if (a >= ring_lo) {
            int64_t const pos = a % S;
            e = std::min<int64_t>(b, a - pos + S);
            g.kind = kGrabRing;
            g.src = (uint64_t)(uintptr_t)ch->d_ring.p + (uint64_t)s * kGrabRingBytes + (uint64_t)pos;
        } else if (a >= c0) {
            e = std::min<int64_t>(b, ring_lo);
            g.kind = kGrabBatch;
            g.src = ctx->offsets[s] + (uint64_t)(a - c0);
        } else {
            e = std::min<int64_t>(std::min<int64_t>(b, c0), ring_lo);
            g.kind = kGrabPrior;
            g.src = ch->pre_off[s] + (uint64_t)(a - (int64_t)ch->pre_lo[s]);
        }
        g.len = (uint64_t)(e - a);
        seg_stream.push_back(g.kind == kGrabBatch ? s : UINT32_MAX);
        segs.push_back(g);
        dst += g.len;
        a = e;
    }
}

// k_grab over `segs` (covering [0, total)) into `out` (device, total rounded up to kGrabSpan); the batch's bytes are
// read from `batch` with `flip`
int grab_launch(r433b_ctx *ctx, std::vector<GrabSeg> const &segs, uint64_t total, uint8_t const *batch, unsigned flip,
        uint8_t const *prior, void *out)
{
    cudaStream_t const st = 0;
    if (int r = dev_reserve(ctx, ctx->d_grab_segs, segs.size() * sizeof(GrabSeg))) return r;
    CU(cudaMemcpyAsync(ctx->d_grab_segs.p, segs.data(), segs.size() * sizeof(GrabSeg), cudaMemcpyHostToDevice, st));
    GrabParams gp{};
    gp.batch = batch;
    gp.prior = prior;
    gp.segs = (GrabSeg const *)ctx->d_grab_segs.p;
    gp.n_segs = (unsigned)segs.size();
    gp.flip = flip;
    gp.total = total;
    gp.out = (uint4 *)out;
    uint64_t const warps = (total + kGrabSpan - 1) / kGrabSpan;
    unsigned const grid = (unsigned)((warps * 32 + kGrabThreads - 1) / kGrabThreads);
    R4_LAUNCH(k_grab, grid, kGrabThreads, 0, st, gp);
    CU(cudaGetLastError());
    return R433B_OK;
}

// k_grab over `segs` (covering [0, total)) into the staging buffer, then one copy to `out`.  In a mixed batch the
// streams' bytes lie in two buffers (the caller's, the converted cf32 streams') and cs8 alone is flipped: one k_grab per
// (buffer, flip) gathers its segments into a region of its own, and the host puts every segment in its place.
int grab_gather(r433b_ctx *ctx, std::vector<GrabSeg> const &segs, std::vector<uint32_t> const &seg_stream, uint64_t total,
        uint8_t *out)
{
    if (!total) return R433B_OK;
    cudaStream_t const st = 0;
    void const *prior = ctx->chained ? ctx->chain_last->d_pre.p : ctx->d_grab_prior.p;
    if (ctx->mixed.empty()) {
        uint64_t const staged = (total + kGrabSpan - 1) / kGrabSpan * kGrabSpan;
        if (int r = dev_reserve(ctx, ctx->d_grab_stage, staged)) return r;
        CU(cudaEventRecord(ctx->ev[0], st));
        if (int r = grab_launch(ctx, segs, total, ctx->grab_src, ctx->grab_flip, (uint8_t const *)prior, ctx->d_grab_stage.p)) return r;
        CU(cudaEventRecord(ctx->ev[1], st));
        CU(cudaMemcpy(out, ctx->d_grab_stage.p, total, cudaMemcpyDeviceToHost));
        cudaEventElapsedTime(&ctx->timing.grab_ms, ctx->ev[0], ctx->ev[1]);
        return R433B_OK;
    }
    struct Group {
        uint8_t const *src;
        unsigned flip;
        std::vector<GrabSeg> segs; // staging positions relative to the group's region
        uint64_t bytes = 0, at = 0;
    };
    std::vector<Group> groups;
    std::vector<std::pair<uint32_t, uint64_t>> place(segs.size()); // segment -> group, its staging position
    for (size_t i = 0; i < segs.size(); ++i) {
        uint32_t const s = seg_stream[i];
        uint8_t const *src = s == UINT32_MAX ? nullptr : ctx->mixed[s].src;
        unsigned const flip = s == UINT32_MAX ? 0u : ctx->mixed[s].flip;
        size_t g = 0;
        while (g < groups.size() && !(s == UINT32_MAX || (groups[g].src == src && groups[g].flip == flip))) ++g;
        if (g == groups.size()) groups.push_back(Group{src, flip, {}});
        GrabSeg q = segs[i];
        q.dst = groups[g].bytes;
        groups[g].segs.push_back(q);
        groups[g].bytes += q.len;
        place[i] = {(uint32_t)g, q.dst};
    }
    uint64_t staged = 0;
    for (Group &g : groups) {
        g.at = staged;
        staged += (g.bytes + kGrabSpan - 1) / kGrabSpan * kGrabSpan;
    }
    if (int r = dev_reserve(ctx, ctx->d_grab_stage, staged)) return r;
    CU(cudaEventRecord(ctx->ev[0], st));
    for (Group const &g : groups)
        if (int r = grab_launch(ctx, g.segs, g.bytes, g.src, g.flip, (uint8_t const *)prior, (uint8_t *)ctx->d_grab_stage.p + g.at))
            return r;
    CU(cudaEventRecord(ctx->ev[1], st));
    std::vector<uint8_t> host(staged);
    CU(cudaMemcpy(host.data(), ctx->d_grab_stage.p, staged, cudaMemcpyDeviceToHost));
    cudaEventElapsedTime(&ctx->timing.grab_ms, ctx->ev[0], ctx->ev[1]);
    for (size_t i = 0; i < segs.size(); ++i)
        memcpy(out + segs[i].dst, host.data() + groups[place[i].first].at + place[i].second, segs[i].len);
    return R433B_OK;
}

static_assert(kGrabRingBytes == R433B_GRAB_RING, "k_grab_ring's ring size");

// After a grabbing chain's batch: save the ring bytes the append overwrites that the batch's frames may still read
// (k_grab), then append every slot's chunk to its ring (k_grab_ring).  A frame that ends in this batch ends at a block
// call, so it reads its slot's run from the end of the chunk's first block minus the ring size on.  The slots of a mixed
// batch read different buffers with different flips: one k_grab_ring per (buffer, flip), in which the other slots
// append nothing (n = 0 and w0 = 0 give no words, so their warps return at once).
int chain_grab_append_launch(r433b_ctx *ctx, r433b_chain *ch)
{
    try {
        cudaStream_t const st = 0;
        int64_t const S = kGrabRingBytes, B = ctx->batch.block_bytes;
        uint32_t const n = ch->n;
        std::vector<GrabSeg> segs;
        std::vector<GrabRingSlot> slots(n);
        std::vector<uint64_t> pre_lo(n), pre_off(n);
        uint64_t pre = 0, max_words = 0;
        for (uint32_t s = 0; s < n; ++s) {
            int64_t const L = (int64_t)ctx->lengths[s], c0 = (int64_t)ch->run[s], c1 = c0 + L;
            int64_t const lo = std::max<int64_t>(0, c0 + std::min(B, L) - S), hi = std::min(c0, c1 - S);
            pre_lo[s] = (uint64_t)lo;
            pre_off[s] = pre;
            for (int64_t a = lo; a < hi;) { // the ring bytes of [lo, hi), split at the wrap
                int64_t const pos = a % S, e = std::min(hi, a - pos + S);
                GrabSeg g{};
                g.dst = pre;
                g.src = (uint64_t)(uintptr_t)ch->d_ring.p + (uint64_t)s * kGrabRingBytes + (uint64_t)pos;
                g.len = (uint64_t)(e - a);
                g.kind = kGrabRing;
                segs.push_back(g);
                pre += g.len;
                a = e;
            }
            int64_t const m = std::min(L, S);
            slots[s].src = ctx->offsets[s] + (uint64_t)(L - m);
            slots[s].n = (unsigned)m;
            slots[s].w0 = (unsigned)((c1 - m) % S);
            max_words = std::max<uint64_t>(max_words, std::min<uint64_t>(((c1 - m) % 16 + m + 15) / 16, S / 16));
        }
        struct Source {
            uint8_t const *batch;
            unsigned flip;
            std::vector<GrabRingSlot> slots;
            uint64_t max_words;
        };
        std::vector<Source> sources;
        if (ctx->mixed.empty()) {
            sources.push_back(Source{ctx->grab_src, ctx->grab_flip, slots, max_words});
        } else {
            for (uint32_t s = 0; s < n; ++s) {
                r433b_ctx::MixedStream const &m = ctx->mixed[s];
                size_t g = 0;
                while (g < sources.size() && !(sources[g].batch == m.src && sources[g].flip == m.flip)) ++g;
                if (g == sources.size()) sources.push_back(Source{m.src, m.flip, std::vector<GrabRingSlot>(n), 0});
                sources[g].slots[s] = slots[s];
                sources[g].max_words = std::max<uint64_t>(sources[g].max_words, std::min<uint64_t>(
                        (slots[s].w0 % 16 + slots[s].n + 15) / 16, S / 16));
            }
        }
        CU(cudaEventRecord(ctx->ev[0], st));
        if (pre) { // ring bytes only: no batch buffer is read
            if (int r = dev_reserve(ctx, ch->d_pre, (pre + kGrabSpan - 1) / kGrabSpan * kGrabSpan)) return r;
            if (int r = grab_launch(ctx, segs, pre, ctx->grab_src, ctx->grab_flip, nullptr, ch->d_pre.p)) return r;
        }
        for (Source const &src : sources) {
            if (!src.max_words) continue;
            CU(cudaMemcpyAsync(ch->d_ring_slots.p, src.slots.data(), n * sizeof(GrabRingSlot), cudaMemcpyHostToDevice, st));
            GrabRingParams rp{};
            rp.batch = src.batch;
            rp.rings = (uint8_t *)ch->d_ring.p;
            rp.slots = (GrabRingSlot const *)ch->d_ring_slots.p;
            uint64_t const per_cta = kGrabThreads / 32 * (kGrabSpan / 16);
            rp.ctas = (unsigned)((src.max_words + per_cta - 1) / per_cta);
            rp.flip = src.flip;
            R4_LAUNCH(k_grab_ring, n * rp.ctas, kGrabThreads, 0, st, rp);
            CU(cudaGetLastError());
        }
        CU(cudaEventRecord(ctx->ev[1], st));
        CU(cudaEventSynchronize(ctx->ev[1]));
        cudaEventElapsedTime(&ctx->timing.grab_ring_ms, ctx->ev[0], ctx->ev[1]);
        // the rings hold the batch: the slots' runs move on
        for (uint32_t s = 0; s < n; ++s) {
            ch->run_c0[s] = ch->run[s];
            ch->run[s] += ctx->lengths[s];
        }
        ch->pre_lo.swap(pre_lo);
        ch->pre_off.swap(pre_off);
        ch->frame = ch->frame_next;
        ch->counter = ch->counter_next;
        ch->grab_pending = true;
        return R433B_OK;
    } catch (std::exception const &) { // allocation failures of the host vectors
        return fail(ctx, R433B_ENOMEM, "r433b_process_chained: out of host memory");
    }
}

// A failed append leaves the rings out of step with the runs: the chain then refuses to grab rather than grab wrong
int chain_grab_append(r433b_ctx *ctx, r433b_chain *ch)
{
    int const r = chain_grab_append_launch(ctx, ch);
    if (r) ch->grab_failed = true;
    return r;
}

// The block calls of push_sdr_flow() on stream s (src/rtl_433.c:1797-1854, src/r_flow.c:137-147, :245-362): its
// blocks from blk0 on, then the flush when its file ends.  `base` is the run's byte count before the stream's first
// call; f carries the stream's frame in and out, `counter` the run's file counter, k the first package not yet
// replayed.  The grabs that `mode` takes go to ctx->grabs.
void grab_replay(r433b_ctx *ctx, r433b_results const *res, int mode, uint32_t s, uint64_t base, uint64_t blk0,
        bool flush, GrabFrame &f, uint32_t &counter, uint32_t &k)
{
    uint32_t const S = R433B_GRAB_RING;
    uint32_t const SS = stream_format(ctx, s).SS, B = ctx->batch.block_bytes;
    r433b_package const *pk = res->packages;
    uint32_t const n_pk = res->n_packages;
    uint64_t const L = ctx->lengths[s];
    uint64_t const n_blocks = (L + B - 1) / B, calls = n_blocks + (flush ? 1 : 0); // call n_blocks is the flush
    uint32_t first = UINT32_MAX; // the frame's first package in this batch
    while (k < n_pk && pk[k].stream < s) ++k;
    for (uint64_t c = 0; c < calls; ++c) {
        uint64_t const blk = blk0 + c;
        bool const here = k < n_pk && pk[k].stream == s && (uint64_t)pk[k].block == blk;
        if (!f.start_ago && !here) { // no frame and no package: nothing but ageing until the next package
            if (k < n_pk && pk[k].stream == s && (uint64_t)pk[k].block > blk) c = (uint64_t)pk[k].block - blk0 - 1;
            else break;
            continue;
        }
        uint64_t const len = c < n_blocks ? std::min<uint64_t>(B, L - c * B) : 0;
        uint32_t const n_samples = (uint32_t)(len / SS);
        uint64_t const P = base + std::min<uint64_t>(L, c * B + len); // pushed after this call's push
        if (f.start_ago) f.start_ago += n_samples;
        if (f.end_ago) f.end_ago += n_samples;
        for (; k < n_pk && pk[k].stream == s && (uint64_t)pk[k].block == blk; ++k) {
            if (!f.start_ago) {
                f.start_ago = pk[k].start_ago;
                first = k;
            } else if (first == UINT32_MAX)
                first = k;
            f.end_ago = pk[k].end_ago;
            uint32_t const pe = ctx->p_events[k];
            f.events += pe;
            if (mode == R433B_GRAB_UNDECODED && pe == 0) {
                uint32_t const q = (uint32_t)analysis_check(pk[k].num_pulses, ctx->an[ctx->dev_index[k]]);
                if (q > f.quality) f.quality = q;
            }
        }
        if (!(f.start_ago && f.end_ago > n_samples)) continue;
        bool const take = mode == R433B_GRAB_ALL || (mode == R433B_GRAB_UNKNOWN && f.events == 0)
                || (mode == R433B_GRAB_KNOWN && f.events > 0) || (mode == R433B_GRAB_UNDECODED && f.events == 0 && f.quality > 0);
        if (take) {
            // unsigned arithmetic of src/r_flow.c:352-356 and samp_grab_write(), src/samp_grab.c:98-134
            uint32_t const pad = n_samples / 8;
            uint32_t const start_padded = f.start_ago + pad, end_padded = f.end_ago - pad;
            uint32_t const grab_len = start_padded - end_padded;
            uint32_t bsize = SS * grab_len;
            bsize += 131072u - bsize % 131072u;
            uint32_t const sg_len = (uint32_t)std::min<uint64_t>(P, S);
            if (bsize > sg_len) bsize = sg_len;
            uint32_t const sg_index = (uint32_t)(P % S);
            uint32_t end_pos = SS * end_padded;
            end_pos = sg_index >= end_pos ? sg_index - end_pos : S - end_pos + sg_index;
            uint64_t const back = ((uint64_t)sg_index + S - end_pos % S) % S; // bytes between window end and newest
            r433b_grab g{};
            g.stream = s;
            g.first_package = first == UINT32_MAX ? k : first;
            g.n_packages = k - g.first_package;
            g.grab_len = grab_len;
            g.bytes = bsize;
            g.counter = counter++;
            g.run_end = (int64_t)P - (int64_t)back;
            ctx->grabs.push_back(g);
            ctx->grab_newest.push_back((int64_t)P);
        }
        f = GrabFrame{};
        first = UINT32_MAX;
    }
}

} // namespace

extern "C" {

int r433b_grab_plan(r433b_ctx *ctx, r433b_results const *res, int mode, r433b_grab_ring const *prior,
        r433b_grab const **grabs, uint32_t *n)
{
    try {
        if (!ctx || !res || !grabs || !n) return fail(ctx, R433B_EINVAL, "null argument");
        if (mode < R433B_GRAB_ALL || mode > R433B_GRAB_UNDECODED) return fail(ctx, R433B_EINVAL, "grab mode must be 1 .. 4");
        if (prior && prior->pushed && !prior->tail) return fail(ctx, R433B_EINVAL, "prior ring without its tail");
        if (!ctx->fetched) return fail(ctx, R433B_ESTATE, "r433b_grab_plan before r433b_fetch");
        if (ctx->pulse_mode) return fail(ctx, R433B_ESTATE, "a batch of loaded pulse data has no IQ to grab");
        r433b_chain *const ch = ctx->chained ? ctx->chain_last : nullptr;
        if (ctx->chained) {
            if (!ch || !ch->grab_mode)
                return fail(ctx, R433B_ESTATE, "the chain of this batch does not grab (r433b_chain_grab before its files)");
            if (ch->grab_failed)
                return fail(ctx, R433B_ESTATE, "appending this batch to its chain's rings failed");
            if (prior) return fail(ctx, R433B_EINVAL, "a chained batch's plan takes no prior: the chain holds the rings");
            if (mode != ch->grab_mode) return fail(ctx, R433B_EINVAL, "grab mode differs from the chain's");
        }
        if (res->packages != (r433b_package const *)ctx->h_pkgs.p || res->n_packages != ctx->n_pkgs)
            return fail(ctx, R433B_EINVAL, "results are not the context's last fetched batch");
        if (mode != R433B_GRAB_ALL)
            for (uint32_t i = 0; i < res->n_packages; ++i)
                if (!ctx->dispatched[res->packages[i].stream])
                    return fail(ctx, R433B_ESTATE, "grab modes 2-4 need every stream with packages dispatched first");
        if (mode == R433B_GRAB_UNDECODED && !ctx->analyzed)
            return fail(ctx, R433B_ESTATE, "grab mode 4 (undecoded) needs r433b_analyze() first");
        CU(cudaSetDevice(ctx->device));
        uint32_t const n_streams = ctx->batch.n_streams;
        ctx->grabs.clear();
        ctx->grab_newest.clear();
        uint32_t k = 0;
        if (ch) { // every slot is its own run: its frame and counter carry over from the slot's last batch
            uint32_t const B = ctx->batch.block_bytes;
            for (uint32_t s = 0; s < n_streams; ++s) {
                GrabFrame f = ch->frame[s];
                uint32_t counter = ch->counter[s];
                uint64_t const blk0 = ctx->chain_base[s] * stream_format(ctx, s).SS / B;
                grab_replay(ctx, res, mode, s, ch->run_c0[s], blk0, ch->ended[s], f, counter, k);
                ch->frame_next[s] = ch->ended[s] ? GrabFrame{} : f; // reset_sdr_flow()
                ch->counter_next[s] = counter;
            }
            ch->grab_pending = false;
        } else { // one run over the streams in batch order; the frame state is per file (reset_sdr_flow(), src/r_flow.c:79-97)
            uint32_t const S = R433B_GRAB_RING;
            uint64_t const pushed = prior ? prior->pushed : 0;
            uint64_t const tail = std::min<uint64_t>(pushed, S);
            if (int r = dev_reserve(ctx, ctx->d_grab_prior, tail + 16)) return r;
            if (tail) CU(cudaMemcpy(ctx->d_grab_prior.p, prior->tail, tail, cudaMemcpyHostToDevice));
            ctx->grab_pushed = pushed;
            ctx->grab_prior_bytes = tail;
            ctx->grab_cum.assign(n_streams + 1, 0);
            for (uint32_t i = 0; i < n_streams; ++i) ctx->grab_cum[i + 1] = ctx->grab_cum[i] + ctx->lengths[i];
            uint32_t counter = prior ? prior->counter : 1; // samp_grab_create() starts at 1
            for (uint32_t s = 0; s < n_streams; ++s) {
                GrabFrame f{};
                grab_replay(ctx, res, mode, s, pushed + ctx->grab_cum[s], 0, true, f, counter, k);
            }
        }
        ctx->grab_planned = true;
        *grabs = ctx->grabs.data();
        *n = (uint32_t)ctx->grabs.size();
        return R433B_OK;
    } catch (std::exception const &) { // allocation failures of the host vectors
        return fail(ctx, R433B_ENOMEM, "r433b_grab_plan: out of host memory");
    }
}

int r433b_grab_copy(r433b_ctx *ctx, r433b_results const *res, uint32_t first, uint32_t count, uint8_t *out, size_t cap)
{
    try {
        if (!ctx || !res) return fail(ctx, R433B_EINVAL, "null argument");
        if (!ctx->grab_planned || (ctx->chained && !ctx->chain_last))
            return fail(ctx, R433B_ESTATE, "r433b_grab_copy before r433b_grab_plan, or after its chain was destroyed");
        if ((uint64_t)first + count > ctx->grabs.size()) return fail(ctx, R433B_EINVAL, "grab index out of range");
        CU(cudaSetDevice(ctx->device));
        uint64_t dst = 0;
        std::vector<GrabSeg> segs;
        std::vector<uint32_t> seg_stream;
        for (uint32_t i = first; i < first + count; ++i) {
            r433b_grab const &g = ctx->grabs[i];
            auto segments = [&](int64_t a, int64_t b) {
                if (ctx->chained) chain_grab_segments(ctx, ctx->chain_last, g.stream, a, b, dst, segs, seg_stream);
                else grab_segments(ctx, a, b, dst, segs, seg_stream);
            };
            int64_t const lo = g.run_end - (int64_t)g.bytes, hi = g.run_end;
            // positions older than the ring holds read its newest bytes at the same slots (one wrap at most: bytes <= ring)
            int64_t const oldest = ctx->grab_newest[i] - (int64_t)R433B_GRAB_RING;
            if (lo < oldest) {
                segments(lo + (int64_t)R433B_GRAB_RING, std::min<int64_t>(hi, oldest) + (int64_t)R433B_GRAB_RING);
                segments(oldest, hi);
            } else
                segments(lo, hi);
        }
        if (dst > cap || (dst && !out)) return fail(ctx, R433B_EINVAL, "output buffer smaller than the grabs' bytes");
        return grab_gather(ctx, segs, seg_stream, dst, out);
    } catch (std::exception const &) { // allocation failures of the host vectors
        return fail(ctx, R433B_ENOMEM, "r433b_grab_copy: out of host memory");
    }
}

int r433b_grab_tail(r433b_ctx *ctx, r433b_results const *res, uint8_t *tail, uint64_t *pushed)
{
    try {
        if (!ctx || !res || !tail || !pushed) return fail(ctx, R433B_EINVAL, "null argument");
        if (!ctx->grab_planned) return fail(ctx, R433B_ESTATE, "r433b_grab_tail before r433b_grab_plan");
        if (ctx->chained) return fail(ctx, R433B_ESTATE, "a chained batch's rings stay in its chain: no r433b_grab_tail");
        CU(cudaSetDevice(ctx->device));
        int64_t const end = (int64_t)(ctx->grab_pushed + ctx->grab_cum.back());
        int64_t const begin = std::max<int64_t>(0, end - (int64_t)R433B_GRAB_RING);
        uint64_t dst = 0;
        std::vector<GrabSeg> segs;
        std::vector<uint32_t> seg_stream;
        grab_segments(ctx, begin, end, dst, segs, seg_stream);
        *pushed = (uint64_t)end;
        return grab_gather(ctx, segs, seg_stream, dst, tail);
    } catch (std::exception const &) { // allocation failures of the host vectors
        return fail(ctx, R433B_ENOMEM, "r433b_grab_tail: out of host memory");
    }
}

} // extern "C"
