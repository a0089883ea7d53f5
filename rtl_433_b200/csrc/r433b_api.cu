// r433b_api.cu -- the C ABI declared in include/r433b.h: context, batch processing on the GPU,
// result fetch, and the CPU-side replay that feeds events to decoders in the reference's order.
// There is no CPU implementation of the DSP here: every sample goes through k_detect/k_slice2.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <atomic>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/r433b.h"
#include "../../include/r433b_abi.h"
#include "r433b_kernels.cuh"
#include "r433b_host.hpp"
#include "r433b_pulses.hpp"
#include "r433b_analyze.cuh"
#include "r433b_analyze_host.hpp"

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
    unsigned fpdm = 0;
    int enable_fm = 0;
    int n_sms = 132;        // cudaDevAttrMultiProcessorCount of `device`
    int spoil_front = 0; // R433B_SPOIL_FRONT=1|2: k_front starts from wrong guesses (tests of the redo / repair paths)
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
    DevBuf d_order; // k_bucket: package indices sorted by (type, length class), per range
    DevBuf d_ranges, d_state, d_lengths, d_stage, d_raw, d_log, d_amoff, d_chunks;
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
};

struct r433b_pulses {
    PulseSet set;
};

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

int dev_reserve(r433b_ctx *ctx, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return 0;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    size_t want = bytes + bytes / 8 + 256;
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
    for (auto &v : ctx->ev) cudaEventCreate(&v);
    cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_det, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking);
    for (auto &v : ctx->ev_in) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_det) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_slc) cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto &v : ctx->ev_t) cudaEventCreate(&v);
    for (auto &v : ctx->ev_f) cudaEventCreate(&v);
    cudaEventCreateWithFlags(&ctx->ev_init, cudaEventDisableTiming);
    ctx->lv = compute_levels(0, 0.0f, -12.1442f, 9.0f);
    if (char const *v = getenv("R433B_SPOIL_FRONT")) ctx->spoil_front = atoi(v);
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
    for (DevBuf *b : {&ctx->d_data, &ctx->d_offsets, &ctx->d_train, &ctx->d_pkgs, &ctx->d_ppool, &ctx->d_gpool,
                 &ctx->d_counters, &ctx->d_am, &ctx->d_fm, &ctx->d_devparams, &ctx->d_lists, &ctx->d_pairs,
                 &ctx->d_arena, &ctx->d_cursor, &ctx->d_ranges, &ctx->d_state, &ctx->d_lengths, &ctx->d_stage, &ctx->d_raw, &ctx->d_log, &ctx->d_amoff, &ctx->d_chunks,
                 &ctx->d_order, &ctx->d_an, &ctx->d_an_dev, &ctx->d_an_gap, &ctx->d_an_pairs, &ctx->d_an_arena})
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
    for (cudaStream_t st : {ctx->s_in, ctx->s_det, ctx->s_out})
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

// The slicers over one package range: k_bucket sorts its packages, k_slice2 runs every slicer on them with the
// tables of sample rate `rate_index`.  `n_pkgs` bounds the range, whose end may only be known on the device.
void launch_slice(r433b_ctx *ctx, GroupRange *range, unsigned n_pkgs, unsigned rate_index, cudaStream_t st)
{
    unsigned const n_devs = (unsigned)ctx->devs.size();
    r433b_package *pkgs = (r433b_package *)ctx->d_pkgs.p;
    SliceParams q{};
    q.pkgs = pkgs;
    q.range = range;
    q.order = (unsigned const *)ctx->d_order.p;
    q.pulse_pool = (int const *)ctx->d_ppool.p;
    q.gap_pool = (int const *)ctx->d_gpool.p;
    q.dev = (SlicerParams const *)ctx->d_devparams.p + (size_t)rate_index * n_devs;
    q.n_devs = n_devs;
    q.ook_list = (unsigned const *)ctx->d_lists.p;
    q.fsk_list = q.ook_list + ctx->n_ook;
    q.n_ook = ctx->n_ook;
    q.n_fsk = ctx->n_fsk;
    q.pairs = (r433b_pair *)ctx->d_pairs.p;
    q.arena = (uint8_t *)ctx->d_arena.p;
    q.arena_cap = ctx->arena_cap;
    q.cursor = (unsigned long long *)ctx->d_cursor.p;
    q.stage = (uint32_t *)ctx->d_stage.p;
    q.stage_words = kStageWords;
    unsigned const bgrid = (unsigned)ctx->n_sms * 2;
    R4_LAUNCH(k_bucket_count, bgrid, kBucketThreads, 0, st, range, pkgs, n_pkgs, n_devs);
    R4_LAUNCH(k_bucket_scan, 1, 1, 0, st, range);
    R4_LAUNCH(k_bucket_scatter, bgrid, kBucketThreads, 0, st, range, (r433b_package const *)pkgs, n_pkgs, (unsigned *)ctx->d_order.p);
    R4_LAUNCH(k_slice2, (unsigned)ctx->n_sms * kSliceCtasPerSm, kSliceThreads, 0, st, q);
}

// The slicer stage over package ranges known on the host: range g (pkg_begin / pkg_end set, the rest zero) uses
// slicer table g.  Runs again with an event arena grown to what the device counted until every event fits, times
// the stage with ev[2] -> ev[3] and leaves the event totals in the context.
int slice_ranges(r433b_ctx *ctx, std::vector<GroupRange> const &ranges, unsigned n_pkgs, cudaStream_t st)
{
    unsigned const n_devs = (unsigned)ctx->devs.size();
    unsigned long long cursor[4] = {0, 0, 0, 0};
    ctx->timing.slice_launches = 0;
    CU(cudaEventRecord(ctx->ev[2], st));
    if (n_pkgs && n_devs) {
        size_t const pair_bytes = (size_t)n_pkgs * n_devs * sizeof(r433b_pair);
        if (int r = dev_reserve(ctx, ctx->d_pairs, pair_bytes)) return r;
        if (int r = dev_reserve(ctx, ctx->d_order, (size_t)n_pkgs * sizeof(unsigned))) return r;
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
            CU(cudaMemcpyAsync(cursor, ctx->d_cursor.p, sizeof(cursor), cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            if (!cursor[2]) break;
            ctx->arena_cap = (size_t)cursor[0] + (1u << 20);
            if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "event arena overflow");
        }
    }
    CU(cudaEventRecord(ctx->ev[3], st));
    CU(cudaEventSynchronize(ctx->ev[3]));
    cudaEventElapsedTime(&ctx->timing.slice_ms, ctx->ev[2], ctx->ev[3]);
    ctx->event_bytes = cursor[0];
    ctx->n_events = cursor[1];
    ctx->n_gated = cursor[3];
    return R433B_OK;
}

} // namespace

int r433b_process(r433b_ctx *ctx, r433b_batch const *b)
{
    if (!ctx || !b || !b->offsets || (b->n_streams && !b->data)) return fail(ctx, R433B_EINVAL, "null argument");
    if (b->sample_format != R433B_FMT_CU8 && b->sample_format != R433B_FMT_CS16 && b->sample_format != R433B_FMT_CS8
            && b->sample_format != R433B_FMT_CF32)
        return fail(ctx, R433B_EINVAL, "sample_format must be R433B_FMT_CU8, _CS8, _CS16 or _CF32");
    // cf32 becomes cs16 on the device before anything else (src/rtl_433.c:1811-1825): from here on
    // offsets, lengths and byte counts are those of the cs16 stream (half the cf32 ones)
    bool const cf32 = b->sample_format == R433B_FMT_CF32;
    unsigned const in_div = cf32 ? 2 : 1;
    if (b->samp_rate == 0) return fail(ctx, R433B_EINVAL, "samp_rate is 0");
    int const SS = (int)(b->sample_format & 0xff); // bytes per IQ sample; cs8 is cu8 after the load-time +128
    uint32_t block_bytes = b->block_bytes ? b->block_bytes : 262144u;
    int const T = kTile;
    if (block_bytes % (uint32_t)(T * SS) != 0) return fail(ctx, R433B_EINVAL, "block_bytes must be a multiple of 2048 samples (4096 bytes of cu8, 8192 of cs16)");
    for (uint32_t i = 0; i <= b->n_streams; ++i) {
        if (b->offsets[i] % (16 * in_div)) return fail(ctx, R433B_EINVAL, "stream offsets must be multiples of 16 bytes (32 for cf32)");
        if (i && b->offsets[i] < b->offsets[i - 1]) return fail(ctx, R433B_EINVAL, "offsets not ascending");
    }
    CU(cudaSetDevice(ctx->device));
    ctx->processed = ctx->fetched = false;
    ctx->pulse_mode = false;
    ctx->batch = *b;
    ctx->batch.sample_format = (uint32_t)SS; // the host replay only needs the sample size (dm_state.sample_size)
    ctx->batch.block_bytes = block_bytes;
    ctx->offsets.assign(b->offsets, b->offsets + b->n_streams + 1);
    for (auto &v : ctx->offsets) v /= in_div;
    ctx->batch.offsets = ctx->offsets.data();
    ctx->lengths.resize(b->n_streams);
    for (uint32_t i = 0; i < b->n_streams; ++i) {
        uint64_t gap = b->offsets[i + 1] - b->offsets[i];
        ctx->lengths[i] = b->lengths ? b->lengths[i] : gap;
        if (ctx->lengths[i] > gap) return fail(ctx, R433B_EINVAL, "lengths[i] exceeds the gap to the next offset");
        if (cf32) ctx->lengths[i] = ctx->lengths[i] / 8 * 4; // whole IQ pairs of floats -> cs16 bytes
    }
    ctx->batch.lengths = ctx->lengths.data();
    uint64_t const total_bytes = b->n_streams ? b->offsets[b->n_streams] / in_div : 0;
    uint64_t used_bytes = 0;
    for (uint64_t v : ctx->lengths) used_bytes += v;
    uint32_t const n_devs = (uint32_t)ctx->devs.size();

    // src/rtl_433.c:1094-1102 and :1515-1522
    ctx->fpdm = b->fpdm_mode == R433B_FPDM_AUTO ? (b->center_frequency > 800000000u ? 1u : 0u) : b->fpdm_mode;
    ctx->enable_fm = 0;
    for (auto const &d : ctx->devs)
        if (d.modulation >= 16) ctx->enable_fm = 1;

    cudaStream_t const st = 0;
    ctx->d2h_done = false;

    // ---- device buffers and launch parameters (no data moved yet) -----------------------
    uint8_t const *d_in;
    if (b->data_on_device && !cf32) {
        d_in = (uint8_t const *)b->data;
    } else {
        if (int r = dev_reserve(ctx, ctx->d_data, total_bytes + 64)) return r;
        d_in = (uint8_t const *)ctx->d_data.p;
    }
    if (cf32 && !b->data_on_device)
        if (int r = dev_reserve(ctx, ctx->d_raw, 2 * total_bytes + 64)) return r;
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
    if (int r = dev_reserve(ctx, ctx->d_amoff, (b->n_streams + 1) * sizeof(uint64_t))) return r;
    CU(cudaMemcpy(ctx->d_amoff.p, ctx->am_offsets.data(), (b->n_streams + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (b->want_stages)
        if (int r = dev_reserve(ctx, ctx->d_fm, total_bytes / SS * sizeof(int16_t) + 16)) return r;

    DetectParams dp{};
    dp.data = d_in;
    dp.offsets = (unsigned long long const *)ctx->d_offsets.p;
    dp.lengths = (unsigned long long const *)ctx->d_lengths.p;
    dp.n_streams = b->n_streams;
    dp.stream0 = 0;
    dp.stream_end = b->n_streams;
    dp.sample_begin = 0;
    dp.sample_end = ~0ull;
    dp.first_chunk = 1;
    dp.state = nullptr;
    dp.use_mag = ctx->use_mag;
    dp.flip = b->sample_format == R433B_FMT_CS8 ? 0x80808080u : 0u;
    dp.enable_fm = ctx->enable_fm;
    dp.fpdm = (int)ctx->fpdm;
    dp.rate = b->samp_rate;
    dp.block_samples = block_bytes / SS;
    dp.lv = ctx->lv;
    dp.lpf_a1 = ((int)(0.85408 * 32768)) >> 1; // src/baseband.c:151-152
    dp.lpf_b0 = ((int)(0.07296 * 32768)) >> 1;
    dp.fm_a1 = dp.fm_b0 = 0;
    dp.wrap_free = 1;
    if (ctx->enable_fm) {
        float lp = ctx->fm_low_pass != 0.0f ? ctx->fm_low_pass : ctx->fpdm ? 0.2f : 0.1f; // src/r_flow.c:204
        fm_coeffs(SS == 4, b->samp_rate, lp, dp.fm_a1, dp.fm_b0);
        long long unity = SS == 2 ? 16384ll : (1ll << 30);
        dp.wrap_free = dp.fm_a1 >= 0 && dp.fm_b0 >= 0 && (long long)dp.fm_a1 + 2ll * dp.fm_b0 <= unity;
    }
    dp.train_scratch = (int *)ctx->d_train.p;
    dp.log_scratch = (unsigned *)ctx->d_log.p;
    dp.counters = (unsigned *)ctx->d_counters.p;
    dp.am_offsets = (unsigned long long const *)ctx->d_amoff.p;
    dp.am = (int16_t *)ctx->d_am.p;
    dp.chunks = (ChunkInfo const *)ctx->d_chunks.p;
    dp.want_stages = b->want_stages ? 1 : 0;
    dp.fm_out = b->want_stages ? (int16_t *)ctx->d_fm.p : nullptr;

    uint64_t max_samples = 0;
    for (uint32_t i = 0; i < b->n_streams; ++i) max_samples = std::max<uint64_t>(max_samples, ctx->lengths[i] / SS);
    // k_front over the tiles [sample_begin, sample_end) of every stream, then the walk over the same range
    auto launch_detect = [&](DetectParams const &q, cudaStream_t s, cudaEvent_t after_front) {
        unsigned n = q.stream_end - q.stream0;
        if (!n) return;
        uint64_t const t_end = (std::min<uint64_t>(q.sample_end, max_samples) + T - 1) / T, t_begin = q.sample_begin / T;
        if (t_end > t_begin) {
            FrontParams fp{};
            fp.data = q.data;
            fp.offsets = q.offsets;
            fp.lengths = q.lengths;
            fp.am_offsets = q.am_offsets;
            fp.n_streams = q.n_streams;
            fp.tile_begin = t_begin;
            fp.tiles = (unsigned)(t_end - t_begin);
            fp.use_mag = q.use_mag;
            fp.flip = q.flip;
            fp.block_samples = q.block_samples;
            fp.a1 = q.lpf_a1;
            fp.b0 = q.lpf_b0;
            fp.am = q.am;
            fp.chunks = (ChunkInfo *)ctx->d_chunks.p;
            fp.counters = q.counters;
            fp.spoil = ctx->spoil_front;
            uint64_t const warps = (uint64_t)q.n_streams * fp.tiles;
            unsigned const fgrid = (unsigned)((warps + kFrontWarps - 1) / kFrontWarps);
            void (*ffn)(FrontParams) = SS == 2 ? k_front<2> : k_front<4>;
            size_t const fsm = (size_t)kFrontWarps * (SS == 2 ? FrontStage<2>::kBytes : FrontStage<4>::kBytes);
            R4_LAUNCH(ffn, fgrid, kFrontWarps * 32, fsm, s, fp);
        }
        cudaEventRecord(after_front, s);
        unsigned grid = (n + kDetectWarps - 1) / kDetectWarps;
        size_t sm = (size_t)kDetectWarps * sizeof(WarpSmem);
        void (*kfn)(DetectParams) = SS == 2 ? k_detect<2> : k_detect<4>;
        R4_LAUNCH(kfn, grid, kDetectWarps * 32, sm, s, q);
    };

    // slicer parameters: per device, scaled to this batch's sample rate on the host
    if (int r = upload_slicer_tables(ctx, std::vector<uint32_t>{b->samp_rate}, st)) return r;

    if (ctx->pkg_cap < (size_t)b->n_streams * 16 + 1024) ctx->pkg_cap = (size_t)b->n_streams * 16 + 1024;
    if (ctx->pool_cap < ctx->pkg_cap * 128) ctx->pool_cap = ctx->pkg_cap * 128;
    if (ctx->arena_cap < total_bytes / 2 + (1u << 20)) ctx->arena_cap = total_bytes / 2 + (1u << 20);


    // ---- pipelined path: host input cut into G TIME SLICES of every stream; the copy-in of slice
    //      k+1 and the copy-out of finished ranges overlap the kernels of slice k (three streams).
    //      detect(k) and slice(k) stay on ONE stream: both are issue-bound, running them
    //      concurrently only makes each slower (measured).  (Cutting by streams instead does not help: a warp needs the same
    //      wall time for its stream however few other warps run.)  Detector / filter state is
    //      carried between launches in `StreamState`; results are identical to one launch. ----
    int G = ctx->pipeline_groups;
    uint64_t stride = b->n_streams ? ctx->offsets[1] - ctx->offsets[0] : 0;
    bool uniform = b->n_streams > 0 && stride > 0;
    // one strided copy per time slice needs the streams on a uniform stride; their LENGTHS may differ (capture files of
    // different sizes padded to a common stride): the kernels stop at every stream's own end
    for (uint32_t i = 0; uniform && i < b->n_streams; ++i)
        if (ctx->offsets[i + 1] - ctx->offsets[i] != stride) uniform = false;
    if (G == 0) { // slice size (tools/e2e_sweep.py sweeps it): many slices of >= 128 KiB per stream for cu8 (4096 streams);
                  // cs16 batches (1024 x 4 MiB, FM on: every launch pays the slowest stream's bursts) want >= 512 KiB
        uint64_t const min_slice = SS == 4 ? (512u << 10) : (128u << 10);
        G = (total_bytes >= (256ull << 20) && stride >= (1u << 20)) ? (int)std::min<uint64_t>(r433b_ctx::kMaxGroups, stride / min_slice) : 1;
    }
    if (b->data_on_device && ctx->pipeline_groups == 0) G = 1; // device input: slices only when asked for
    if (b->want_stages || !n_devs || !uniform || cf32) G = 1;
    uint64_t slice_samples = 0;
    if (G > 1) {
        uint64_t n_samp = stride / SS;
        uint64_t unit = (uint64_t)T; // slices only have to be tile aligned: block effects use absolute positions
        slice_samples = (n_samp / G + unit - 1) / unit * unit;
        if (slice_samples == 0 || slice_samples >= n_samp) G = 1;
        else G = (int)((n_samp + slice_samples - 1) / slice_samples);
        if (G > r433b_ctx::kMaxGroups) G = 1;
    }
    if (G > 1) {
        using clk = std::chrono::steady_clock;
        auto t_wall0 = clk::now();
        if (int r = dev_reserve(ctx, ctx->d_pkgs, ctx->pkg_cap * sizeof(r433b_package))) return r;
        if (int r = dev_reserve(ctx, ctx->d_order, ctx->pkg_cap * sizeof(unsigned))) return r;
        if (int r = dev_reserve(ctx, ctx->d_ppool, ctx->pool_cap * sizeof(int))) return r;
        if (int r = dev_reserve(ctx, ctx->d_gpool, ctx->pool_cap * sizeof(int))) return r;
        size_t const pair_cap_bytes = ctx->pkg_cap * n_devs * sizeof(r433b_pair);
        if (int r = dev_reserve(ctx, ctx->d_pairs, pair_cap_bytes)) return r;
        if (int r = dev_reserve(ctx, ctx->d_arena, ctx->arena_cap)) return r;
        if (int r = dev_reserve(ctx, ctx->d_ranges, G * sizeof(GroupRange))) return r;
        if (int r = dev_reserve(ctx, ctx->d_state, (size_t)b->n_streams * sizeof(StreamState))) return r;
        if (int r = host_reserve(ctx, ctx->h_ranges, G * sizeof(GroupRange))) return r;
        dp.pkgs = (r433b_package *)ctx->d_pkgs.p;
        dp.pkg_cap = (unsigned)std::min<size_t>(ctx->pkg_cap, 0xffffffffu);
        dp.pulse_pool = (int *)ctx->d_ppool.p;
        dp.gap_pool = (int *)ctx->d_gpool.p;
        dp.pool_cap = (unsigned)std::min<size_t>(ctx->pool_cap, 0xffffffffu);
        dp.state = (StreamState *)ctx->d_state.p;
        GroupRange *d_rg = (GroupRange *)ctx->d_ranges.p;
        GroupRange *h_rg = (GroupRange *)ctx->h_ranges.p;
        unsigned const *d_cnt = (unsigned const *)ctx->d_counters.p;
        unsigned long long const *d_cur = (unsigned long long const *)ctx->d_cursor.p;

        // the table uploads above went through the legacy stream from pageable memory: their DMA may still be
        // in flight when cudaMemcpy returns, and s_det does not synchronise with stream 0 by itself
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
            launch_detect(dg, ctx->s_det, ctx->ev_f[g]);
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
            size_t pk_hi = (size_t)r.pkg_end * sizeof(r433b_package), pool_hi = (size_t)r.pool_end * sizeof(int);
            size_t pair_hi = (size_t)r.pkg_end * n_devs * sizeof(r433b_pair);
            // the same sizes r433b_fetch() reserves (+16): a buffer that passes here is never reallocated there
            if (ctx->h_pkgs.cap < pk_hi + 16 || ctx->h_ppool.cap < pool_hi + 16 || ctx->h_gpool.cap < pool_hi + 16
                    || ctx->h_pairs.cap < pair_hi + 16 || ctx->h_events.cap < r.arena_end + 16)
                d2h_ok = false;
            if (!d2h_ok) continue;
            size_t pk_lo = (size_t)r.pkg_begin * sizeof(r433b_package), pool_lo = (size_t)r.pool_begin * sizeof(int);
            size_t pair_lo = (size_t)r.pkg_begin * n_devs * sizeof(r433b_pair);
            cudaStream_t so = ctx->s_out;
            if (pk_hi > pk_lo) CU(cudaMemcpyAsync((char *)ctx->h_pkgs.p + pk_lo, (char *)ctx->d_pkgs.p + pk_lo, pk_hi - pk_lo, cudaMemcpyDeviceToHost, so));
            if (pool_hi > pool_lo) {
                CU(cudaMemcpyAsync((char *)ctx->h_ppool.p + pool_lo, (char *)ctx->d_ppool.p + pool_lo, pool_hi - pool_lo, cudaMemcpyDeviceToHost, so));
                CU(cudaMemcpyAsync((char *)ctx->h_gpool.p + pool_lo, (char *)ctx->d_gpool.p + pool_lo, pool_hi - pool_lo, cudaMemcpyDeviceToHost, so));
            }
            if (pair_hi > pair_lo) CU(cudaMemcpyAsync((char *)ctx->h_pairs.p + pair_lo, (char *)ctx->d_pairs.p + pair_lo, pair_hi - pair_lo, cudaMemcpyDeviceToHost, so));
            if (r.arena_end > r.arena_begin)
                CU(cudaMemcpyAsync((char *)ctx->h_events.p + r.arena_begin, (char *)ctx->d_arena.p + r.arena_begin, r.arena_end - r.arena_begin, cudaMemcpyDeviceToHost, so));
        }
        CU(cudaStreamSynchronize(ctx->s_out));
        if (!overflow) {
            GroupRange const last = h_rg[G - 1];
            if ((uint64_t)last.pkg_end * n_devs > 0xffffffffull)
                return fail(ctx, R433B_EOVERFLOW, "packages x devices exceeds the 32-bit pair index (r433b_package.first_pair)");
            ctx->n_pkgs = last.pkg_end;
            ctx->pool_used = last.pool_end;
            ctx->event_bytes = last.arena_end;
            ctx->n_events = last.events_end;
            ctx->n_gated = last.gated_end;
            ctx->n_samples = used_bytes / SS;
            ctx->d2h_done = d2h_ok;
            float det = 0, slc = 0, frt = 0;
            for (int g = 0; g < G; ++g) {
                float a = 0, c = 0, f = 0;
                cudaEventElapsedTime(&f, ctx->ev_t[4 * g + 0], ctx->ev_f[g]);
                cudaEventElapsedTime(&a, ctx->ev_f[g], ctx->ev_t[4 * g + 1]);
                cudaEventElapsedTime(&c, ctx->ev_t[4 * g + 2], ctx->ev_t[4 * g + 3]);
                frt += f;
                det += a;
                slc += c;
            }
            ctx->timing.front_ms = frt;
            ctx->timing.front_launches = (unsigned)G;
            unsigned stat[8];
            CU(cudaMemcpy(stat, ctx->d_counters.p, sizeof(stat), cudaMemcpyDeviceToHost));
            ctx->timing.front_redone = stat[4];
            ctx->timing.front_repairs = stat[5];
            ctx->timing.h2d_ms = 0; // overlapped: only the wall total is meaningful
            ctx->timing.d2h_ms = 0;
            ctx->timing.detect_ms = det;
            ctx->timing.slice_ms = slc;
            ctx->timing.total_ms = std::chrono::duration<float, std::milli>(clk::now() - t_wall0).count();
            ctx->timing.detect_launches = (unsigned)G;
            ctx->timing.slice_launches = (unsigned)G;
            ctx->processed = true;
            return R433B_OK;
        }
        // an arena was too small: grow from what the device counted and redo sequentially below
        unsigned cnt[4];
        unsigned long long cur[4];
        CU(cudaMemcpy(cnt, ctx->d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(cur, ctx->d_cursor.p, sizeof(cur), cudaMemcpyDeviceToHost));
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)cnt[0] * 2 + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)cnt[1] * 2 + 4096);
        ctx->arena_cap = std::max<size_t>(ctx->arena_cap, (size_t)cur[0] * 2 + (1u << 20));
    }

    // ---- sequential path ------------------------------------------------------------------
    CU(cudaEventRecord(ctx->ev[0], st));
    if (cf32 && total_bytes) {
        void const *raw = b->data;
        if (!b->data_on_device) {
            CU(cudaMemcpyAsync(ctx->d_raw.p, b->data, 2 * total_bytes, cudaMemcpyHostToDevice, st));
            raw = ctx->d_raw.p;
        }
        size_t n4 = (size_t)(2 * total_bytes / 16); // groups of four floats (offsets are multiples of 32 bytes)
        R4_LAUNCH(k_cf32_to_cs16, ctx->n_sms * 8, 256, 0, st, (float4 const *)raw, (uint2 *)ctx->d_data.p, n4);
        CU(cudaGetLastError());
    } else if (!b->data_on_device && total_bytes)
        CU(cudaMemcpyAsync(ctx->d_data.p, b->data, total_bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ctx->ev[1], st));

    unsigned detect_launches = 0;
    unsigned counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int attempt = 0; attempt < 3; ++attempt) {
        if (int r = dev_reserve(ctx, ctx->d_pkgs, ctx->pkg_cap * sizeof(r433b_package))) return r;
        if (int r = dev_reserve(ctx, ctx->d_ppool, ctx->pool_cap * sizeof(int))) return r;
        if (int r = dev_reserve(ctx, ctx->d_gpool, ctx->pool_cap * sizeof(int))) return r;
        dp.pkgs = (r433b_package *)ctx->d_pkgs.p;
        dp.pkg_cap = (unsigned)std::min<size_t>(ctx->pkg_cap, 0xffffffffu);
        dp.pulse_pool = (int *)ctx->d_ppool.p;
        dp.gap_pool = (int *)ctx->d_gpool.p;
        dp.pool_cap = (unsigned)std::min<size_t>(ctx->pool_cap, 0xffffffffu);
        CU(cudaMemsetAsync(ctx->d_counters.p, 0, 64, st));
        if (b->n_streams) {
            launch_detect(dp, st, ctx->ev[4]);
            CU(cudaGetLastError());
            detect_launches++;
        }
        CU(cudaMemcpyAsync(counters, ctx->d_counters.p, sizeof(counters), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (!counters[2]) break;
        // arenas were too small: the counters hold the true need
        ctx->pkg_cap = std::max<size_t>(ctx->pkg_cap, (size_t)counters[0] + 64);
        ctx->pool_cap = std::max<size_t>(ctx->pool_cap, (size_t)counters[1] + 4096);
        if (attempt == 2) return fail(ctx, R433B_EOVERFLOW, "package arena overflow");
    }
    if ((uint64_t)counters[0] * n_devs > 0xffffffffull)
        return fail(ctx, R433B_EOVERFLOW, "packages x devices exceeds the 32-bit pair index (r433b_package.first_pair)");
    ctx->n_pkgs = counters[0];
    ctx->pool_used = counters[1];
    GroupRange all{};
    all.pkg_end = ctx->n_pkgs;
    if (int r = slice_ranges(ctx, std::vector<GroupRange>{all}, ctx->n_pkgs, st)) return r;
    ctx->n_samples = used_bytes / SS;
    cudaEventElapsedTime(&ctx->timing.h2d_ms, ctx->ev[0], ctx->ev[1]);
    ctx->timing.front_ms = 0;
    if (detect_launches) {
        cudaEventElapsedTime(&ctx->timing.front_ms, ctx->ev[1], ctx->ev[4]);
        cudaEventElapsedTime(&ctx->timing.detect_ms, ctx->ev[4], ctx->ev[2]);
    } else
        cudaEventElapsedTime(&ctx->timing.detect_ms, ctx->ev[1], ctx->ev[2]);
    ctx->timing.front_launches = detect_launches;
    ctx->timing.front_redone = counters[4];
    ctx->timing.front_repairs = counters[5];
    cudaEventElapsedTime(&ctx->timing.total_ms, ctx->ev[0], ctx->ev[3]);
    ctx->timing.d2h_ms = 0;
    ctx->timing.detect_launches = detect_launches;
    ctx->processed = true;
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
    size_t pk_bytes = (size_t)ctx->n_pkgs * sizeof(r433b_package);
    size_t pool_bytes = (size_t)ctx->pool_used * sizeof(int);
    size_t pair_bytes = (size_t)ctx->n_pkgs * n_devs * sizeof(r433b_pair);
    CU(cudaEventRecord(ctx->ev[4], st));
    if (int r = host_reserve(ctx, ctx->h_pkgs, pk_bytes + 16)) return r;
    if (int r = host_reserve(ctx, ctx->h_ppool, pool_bytes + 16)) return r;
    if (int r = host_reserve(ctx, ctx->h_gpool, pool_bytes + 16)) return r;
    if (int r = host_reserve(ctx, ctx->h_pairs, pair_bytes + 16)) return r;
    if (int r = host_reserve(ctx, ctx->h_events, ctx->event_bytes + 16)) return r;
    if (!ctx->d2h_done) {
        if (pk_bytes) CU(cudaMemcpyAsync(ctx->h_pkgs.p, ctx->d_pkgs.p, pk_bytes, cudaMemcpyDeviceToHost, st));
        if (pool_bytes) {
            CU(cudaMemcpyAsync(ctx->h_ppool.p, ctx->d_ppool.p, pool_bytes, cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(ctx->h_gpool.p, ctx->d_gpool.p, pool_bytes, cudaMemcpyDeviceToHost, st));
        }
        if (pair_bytes && ctx->d_pairs.p) CU(cudaMemcpyAsync(ctx->h_pairs.p, ctx->d_pairs.p, pair_bytes, cudaMemcpyDeviceToHost, st));
        if (ctx->event_bytes) CU(cudaMemcpyAsync(ctx->h_events.p, ctx->d_arena.p, ctx->event_bytes, cudaMemcpyDeviceToHost, st));
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
    uint64_t SS = ctx->batch.sample_format;
    uint64_t bytes = ctx->lengths[k.stream];
    uint32_t bb = ctx->batch.block_bytes;
    uint64_t n_blocks = (bytes + bb - 1) / bb;
    if (n_blocks == 0) return 0.0f;
    // src/rtl_433.c:1839: value set before the block that returned the package was pushed;
    // the flush keeps the last block's value
    uint64_t blk = (uint64_t)k.block < n_blocks ? (uint64_t)k.block : n_blocks - 1;
    unsigned long n_read = (unsigned long)std::min<uint64_t>(bb, bytes - blk * bb);
    float pos = ((float)(int)blk * bb + n_read) / ctx->batch.samp_rate / (int)SS;
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
    pd->offset = k.offset;
    pd->sample_rate = ctx->batch.samp_rate;
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
    uint32_t rate = ctx->batch.samp_rate, center = ctx->batch.center_frequency;
    float off1 = (float)pd->fsk_f1_est / INT16_MAX * rate / 2.0f;
    float off2 = (float)pd->fsk_f2_est / INT16_MAX * rate / 2.0f;
    pd->freq1_hz = off1 + center;
    pd->freq2_hz = off2 + center;
    pd->centerfreq_hz = center;
    pd->depth_bits = ctx->batch.sample_format * 4;
    if (ctx->batch.sample_format == 2 && !ctx->use_mag) {
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
    }
    return R433B_OK;
}

} // namespace

extern "C" {

// Position-independent checksum of everything the batch holds for one stream: package headers (without the
// fields that say where in the batch they lie), pulse and gap widths, and the event bytes of every
// (package, device) pair in device order.  Two streams with the same samples give the same digest wherever
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
            mix(pr.bytes);
            mix(pr.events);
            mix(pr.gated_single);
            mix(pr.gated_multi);
            if (pr.bytes) mix_words(res->events + pr.offset, pr.bytes / 4);
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
    if ((uint64_t)n * n_devs > 0xffffffffull)
        return fail(ctx, R433B_EOVERFLOW, "packages x devices exceeds the 32-bit pair index (r433b_package.first_pair)");
    ctx->processed = ctx->fetched = false;
    ctx->d2h_done = false;
    ctx->pulse_mode = true;
    ctx->pulse_meta = set.pk;
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
        if (ctx->arena_cap < (size_t)(1u << 20)) ctx->arena_cap = 1u << 20;
        if (int r = upload_slicer_tables(ctx, rates, st)) return r;
        if (int r = slice_ranges(ctx, ranges, n, st)) return r;
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
    return ctx->batch.samp_rate;
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
