// r433b_detect.cuh -- k_detect: IQ -> packages, one WARP per capture stream (sm_90a).
//
// The AM (envelope + low-pass) of every sample was made by k_front (r433b_front.cuh), tile-parallel, and lies
// in HBM as 16 bits per sample with the bounds of every 64-sample chunk.  The warp walks its stream in tiles
// of 2048 samples.  Per tile:
//
//  1. Hand-over check.  k_front started every tile but the first of a stream from a GUESS of the filter state.
//     The filter state is its own last output, so the tile fits its predecessor iff
//     step(last AM of the previous tile, x[-1], x[0]) equals the first stored AM of this one.  If not (rare),
//     the walk recomputes forward from the exact state until its values meet the stored ones again; from
//     there on the stored values are the exact ones (k_front's chunks are consistent with each other).
//     In IDLE, whole noise tiles are ruled out from k_front's tile summaries before any of this (idle_skip):
//     their AM is never loaded.
//
//  2. The package detector (src/pulse_detect.c:199-483) walks the tile warp-uniformly with ballot scans for
//     the states whose thresholds are frozen (IDLE stretches by bracket rounds, GAP, GAP_START) and a
//     sequential but lean recurrence for the high-level estimator of PULSE.
//
//  3. FM (src/baseband.c:181-366) is only READ in two places: by the FSK sub-detector during the first
//     pulse of a package, and by the carrier estimate `fsk_f1_est`, which is reported when a package ends.
//     Neither needs FM for every sample:
//       * FM WINDOWS of 256 samples are made on demand (discriminator lane-parallel from the IQ bytes,
//         low-pass by sub-chunks with the same start-from-a-guess / verify / redo scheme).  A window that does
//         not continue the previous one closely gets its filter state rebuilt RIGOROUSLY when the filter is
//         monotone (the host proves a1, b0 >= 0, a1 + 2 b0 <= unity): both ends of the whole state range are
//         pushed through the samples in front of the window until they meet.  Otherwise the walk reads FM
//         in order only, and the windows in between are made from the last exact state.  The stage dump
//         (FM of every sample) is a pass of its own after the walk.
//       * the carrier estimate g' = g + f/64 - g/64 is DEFERRED after the first pulse: the walk only logs
//         which samples update it.  When the package ends, g is evaluated over the newest ~1000 logged
//         samples from both ends of its range; the recurrence forgets its start at 63/64 per sample, the two
//         ends meet, and a met pair is the exact value.  If they do not meet (exactly constant input), the
//         evaluation goes further back, in the end over the whole log from the exactly known value after
//         the first pulse.  A full log is folded into that value the same way.
//
// HBM traffic per sample: IQ once and AM once in k_front, AM once here (plus the IQ of the FM windows).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/r433b.h"
#include "r433b_core.cuh"
#include "r433b_front.cuh"

namespace r433b {

constexpr int kTrainInts = 4 * kMaxPulses; // per-stream scratch: ook pulse/gap, fsk pulse/gap
constexpr int kDetectWarps = 4;            // warps (streams) per CTA
constexpr int kDetectCtasPerSm = 8;        // 32 warps per SM (64 registers): 4096 streams are co-resident on 132 SMs
// R433B_SPLIT_AUTO (r433b_set_split): a batch of fewer streams than resident k_detect warps splits the streams of at least
// kSplitMinSegments segments of at least kSplitMinSegmentBlocks blocks, the segments sized for about one slot per warp
constexpr int kSplitMinSegments = 4;
constexpr int kSplitMinSegmentBlocks = 2;

constexpr int kAmStride = kChunk / 2 + 1;  // words between lane chunks of the 16-bit AM tile (odd: conflict-free)
constexpr int kAmWords = 32 * kAmStride;
constexpr int kFmWin = 256;                // FM window
constexpr int kFmSub = kFmWin / 32;        // samples per lane of a window
constexpr int kFmPadded = kFmWin + kFmWin / kFmSub; // padded index space: i + i / kFmSub
constexpr int kWarmFm = 48;                // warm-up samples of the FM trajectories
constexpr unsigned kLogCap = 1024;         // deferred carrier-estimate log: entries per stream
#ifndef R4_F1_TAIL
#define R4_F1_TAIL 1024
#endif
constexpr int kF1Tail = R4_F1_TAIL;        // samples of the first evaluation attempt; when the two ends have not met, the next
                                           // attempt takes four times as many.  k_detect, 4096 x 2^20 cu8: 768 -> 18.0 ms,
                                           // 1024 -> 17.7, 1280 -> 18.4, 1536 -> 19.0, 2048 -> 20.2; 640 and less: 20+ (retries)

struct FmJob {
    uint8_t const *src;        // the stream
    unsigned long long N;      // its length in samples
    long long a1, b0;
    int16_t *fm_out;           // stage dump (indexed by sample) or nullptr; the walk's is always nullptr
    unsigned flip;
    int fm_on;                 // 0: "FM" is the raw envelope (buf.fm aliases buf.temp when nothing asks for FM)
    int use_mag;
    int monotone;              // the state rebuild by range collapse is valid
    FmState start;             // the exact state in front of sample 0 (reset state, or carried into a chained chunk)
    int pri0, prq0;            // the IQ sample in front of sample 0 (centred; zero at a file start)
};

// Warp-uniform state of the walk.  It lives in shared memory BETWEEN the phases of the walk (idle_run, burst_run,
// generic_step, walk_emit: separate functions, each with the registers and the instruction footprint of its own
// loop); a phase loads what it needs into registers, every lane computes the same values, lane 0 stores them back.
struct WalkState {
    DetState d;
    unsigned log_n, log_start, log_count; // deferred carrier-estimate log: closed entries (global memory), the open entry
    unsigned seq;
    int pend_type;               // a finished package to hand over (1 OOK, 2 FSK) ...
    int skip_y;                  // idle_skip: the AM filter state in front of the tile it returns
    unsigned long long pend_pos; // ... returned at this stream position
    unsigned long long t0;       // the tile being walked
    int nv_tile;
    unsigned rewalk_end;         // idle_skip: tiles (index) in front of this one are walked without skipping (a run walked again)
};

// Per-stream constants of the walk (written once by lane 0)
struct WalkConst {
    FmJob jb;
    Trains tr;
    unsigned *log;
    Levels lv;
    int per_ms, fpdm, defer_f1;
    unsigned stream, block_samples;
    unsigned long long base;     // absolute sample index of sample 0 (chained chunks): added to reported positions
    r433b_package *pkgs;
    int *pulse_pool, *gap_pool;
    unsigned pkg_cap, pool_cap;
    DetectCounters *counters;
    TileInfo const *tiles;       // the stream's tile summaries; nullptr: no tile is skipped (idle_skip)
};

// Shared memory of one warp
struct alignas(16) WarpSmem {
    uint32_t am[kAmWords];       // AM tile, 16 bits per sample: sample n at u16 (n / 64) * 66 + n % 64
    uint32_t xf[kFmPadded];      // discriminator outputs of the current FM window (padded index)
    uint16_t fm[kFmPadded];      // FM (or the raw-envelope alias) of the current window
    int q[32];                   // chain operands of one 32-sample step
    int cmin[32], cmax[32];      // per lane chunk: bounds of its AM values
    // FM bookkeeping (warp-uniform; written by lane 0)
    FmState fm_state;
    unsigned long long win0;     // the window holds FM of [win0, win0 + win_n)
    int win_n;
    WalkState ws;
    WalkConst wc;
};

struct DetectParams {
    uint8_t const *data;
    unsigned long long const *offsets; // bytes, n_streams + 1
    unsigned long long const *lengths; // optional: bytes of stream i actually used
    unsigned long long const *am_offsets; // first sample of stream i in `am` (k_front's output)
    unsigned n_streams;
    unsigned stream0, stream_end;      // the streams this launch covers
    unsigned long long sample_begin, sample_end; // the slice of every stream this launch covers (multiples of the tile)
    int first_chunk;                   // the first launch of the batch: start from reset_sdr_flow() state instead of the
                                       // saved one, except for the streams `cont` marks
    struct StreamState *state;         // per-stream carried state between launches (and chained batches)
    unsigned char const *cont;         // chained: 1 = the stream continues a file, its first launch loads state[s]
    unsigned char const *last;         // chained: 1 = the file ends with this chunk (flush); nullptr: every file ends
    unsigned long long const *base;    // chained: absolute sample index of each stream's sample 0 (nullptr: 0)
    int use_mag, enable_fm, fpdm;
    unsigned flip; // XOR mask applied to every loaded word: 0x80808080 turns cs8 into cu8
    unsigned rate, block_samples;
    Levels lv;
    int lpf_a1, lpf_b0, fm_a1, fm_b0;
    int wrap_free;
    int *train_scratch;
    unsigned *log_scratch;             // n_streams * kLogCap * 2
    r433b_package *pkgs;
    unsigned pkg_cap;
    int *pulse_pool, *gap_pool;
    unsigned pool_cap;
    DetectCounters *counters;
    int16_t *am;               // k_front's output (repaired in place where a tile did not fit its predecessor)
    ChunkInfo const *chunks;   // bounds of every 64-sample chunk of `am`
    TileInfo const *tile_info; // summary of every tile of `am` (as k_front made it: never updated by a repair)
    int16_t *fm_out;           // optional stage dump, indexed by offsets[s]/SS + n (one launch over whole streams)
};

struct WarpCtx {
    int lane;
    int nlanes;
    __device__ __forceinline__ void sync() { __syncwarp(); }
};

__device__ __forceinline__ int fm_pidx(int i) { return i + i / kFmSub; }

// ------------------------------------------------------------------------------ FM --------

// IQ of one sample (centred) out of a loaded group
template <int SS>
__device__ __forceinline__ void iq_of(uint32_t const (&rw)[4], int j, int &ci, int &cq)
{
    if (SS == 2) {
        uint32_t w = rw[j >> 1] >> ((j & 1) * 16);
        ci = (int)(w & 0xff) - 128;
        cq = (int)((w >> 8) & 0xff) - 128;
    } else {
        uint32_t w = rw[j & 3];
        ci = (int)(int16_t)(w & 0xffff);
        cq = (int)(int16_t)(w >> 16);
    }
}

// one low-pass step of the FM filter (src/baseband.c:263 / :357); the cu8 state is an int16 store
template <int SS>
__device__ __forceinline__ int fm_step(int y, long long a1, long long b0, int v, int vp)
{
    if (SS == 2) return iir16(y, (int)a1, (int)b0, v + vp);
    return iir32(y, a1, b0, (long long)v + vp);
}


// Discriminator outputs (src/baseband.c:253-262 / :346-356) of samples [a, a + n) into sm.xf[fm_pidx(i)],
// n <= kFmWin, a a multiple of SPL; lane j of a batch takes the group at a + 32 * SPL * q + SPL * j.
// With !fm_on the raw envelope goes straight to sm.fm instead.
template <int SS>
__device__ R4_NOINLINE void disc_fill(FmJob const &jb, WarpSmem &sm, unsigned long long a, int n)
{
    constexpr int SPL = 16 / SS;
    int const lane = threadIdx.x & 31;
    R4_EMU_ASSERT_POS(a);
    // IQ in front of the batch: at sample 0 the one carried into the chunk (zero at a file start: reset demod state)
    int pri = jb.pri0, prq = jb.prq0;
    if (jb.fm_on && a > 0) iq_at<SS>(jb.src, a - 1, jb.flip, pri, prq);
#pragma unroll 1
    for (int base = 0; base < n; base += 32 * SPL) {
        int const i0 = base + lane * SPL;
        uint32_t rw[4];
        load_group<SS>(jb.src, a + (unsigned long long)i0, i0 < n ? (long long)(jb.N - a) - i0 : 0, jb.flip, rw);
        if (!jb.fm_on) {
            int x[SPL];
            env_group<SS>(rw, jb.use_mag, x);
#pragma unroll
            for (int j = 0; j < SPL; ++j)
                if (i0 + j < n) sm.fm[fm_pidx(i0 + j)] = (uint16_t)x[j];
            continue;
        }
        int li, lq;
        iq_of<SS>(rw, SPL - 1, li, lq);
        int pi_ = __shfl_up_sync(0xffffffffu, li, 1);
        int pq_ = __shfl_up_sync(0xffffffffu, lq, 1);
        if (lane == 0) {
            pi_ = pri;
            pq_ = prq;
        }
        pri = __shfl_sync(0xffffffffu, li, 31);
        prq = __shfl_sync(0xffffffffu, lq, 31);
#pragma unroll
        for (int j = 0; j < SPL; ++j) {
            int ci, cq, xf;
            iq_of<SS>(rw, j, ci, cq);
            if (SS == 2) {
                xf = atan16(cq * pi_ - ci * pq_, ci * pi_ + cq * pq_);
            } else {
                long long re = (long long)ci * pi_ + (long long)cq * pq_;
                long long im = (long long)cq * pi_ - (long long)ci * pq_;
                xf = atan32((int)(unsigned)(unsigned long long)im, (int)(unsigned)(unsigned long long)re);
            }
            pi_ = ci;
            pq_ = cq;
            if (i0 + j < n) sm.xf[fm_pidx(i0 + j)] = (uint32_t)xf;
        }
    }
    __syncwarp();
}

// The exact FM filter state in front of sample `pos` (after sample pos - 1), without knowing anything
// before: both ends of the state range go through the K samples in front of pos; when they meet, the value
// is independent of everything earlier.  K grows until they meet or the walk starts at a known state
// (sample 0, where jb.start holds it, or sm.fm_state.pos).  Monotone filters only.  Leaves the state in sm.fm_state.
template <int SS>
__device__ R4_NOINLINE void fm_cold(FmJob const &jb, WarpSmem &sm, unsigned long long pos)
{
    constexpr int SPL = 16 / SS;
    int const lane = threadIdx.x & 31;
    unsigned long long const known = sm.fm_state.pos; // state known here (always <= pos when used)
    for (unsigned long long K = 64;; K *= 4) {
        unsigned long long a = pos > K ? (pos - K) / SPL * SPL : 0;
        bool exact_start = a == 0;
        int lo, hi, fp;
        if (known <= pos && known >= a) { // reach back to the known state instead
            a = known;
            exact_start = true;
        }
        if (exact_start) {
            lo = hi = a == known ? sm.fm_state.y : jb.start.y;
            fp = a == known ? sm.fm_state.xf : jb.start.xf;
        } else {
            lo = SS == 2 ? -32768 : (int)0x80000000;
            hi = SS == 2 ? 32767 : 0x7fffffff;
            fp = 0; // replaced below by the sample in front of the first processed one
        }
        // pieces of kFmWin samples, sequential chain carried across them
        bool first_piece = true;
        for (unsigned long long p0 = a; p0 < pos; p0 += kFmWin) {
            int const n = pos - p0 < (unsigned long long)kFmWin ? (int)(pos - p0) : kFmWin;
            disc_fill<SS>(jb, sm, p0, n);
            int k = 0;
            if (first_piece && !exact_start) { // the first sample only provides x[n-1]
                fp = (int)sm.xf[fm_pidx(0)];
                k = 1;
            }
            first_piece = false;
#pragma unroll 2
            for (; k < n; ++k) {
                int v = (int)sm.xf[fm_pidx(k)];
                lo = fm_step<SS>(lo, jb.a1, jb.b0, v, fp);
                hi = fm_step<SS>(hi, jb.a1, jb.b0, v, fp);
                fp = v;
            }
            __syncwarp();
        }
        if (lo == hi) {
            if (lane == 0) {
                sm.fm_state = FmState{pos, lo, fp};
                sm.win_n = 0;
            }
            __syncwarp();
            return;
        }
        // not met: exactly constant input parks the two ends on different fixed points of the floor map
    }
}

// FM of the window [w0, w0 + n) (n <= kFmWin, w0 a multiple of SPL) from the exact state in sm.fm_state which
// must be the one in front of w0.  Advances sm.fm_state to w0 + n.
template <int SS>
__device__ R4_NOINLINE void fm_window(FmJob const &jb, WarpSmem &sm, unsigned long long w0, int n)
{
    int const lane = threadIdx.x & 31;
    disc_fill<SS>(jb, sm, w0, n);
    if (jb.fm_on) {
        int const base = lane * kFmSub;
        int nv = n - base;
        nv = nv < 0 ? 0 : (nv > kFmSub ? kFmSub : nv);
        int start = base - kWarmFm;
        bool const exact = start <= 0;
        int y, fp;
        if (exact) {
            start = 0;
            y = sm.fm_state.y;
            fp = sm.fm_state.xf;
        } else {
            fp = (int)sm.xf[fm_pidx(start - 1)];
            y = fp; // the low-pass has unit gain: its state is near its input
        }
        if (nv > 0) {
#pragma unroll 4
            for (int k = start; k < base; ++k) {
                int v = (int)sm.xf[fm_pidx(k)];
                y = fm_step<SS>(y, jb.a1, jb.b0, v, fp);
                fp = v;
            }
        }
        int const y_b = y, fp_b = fp;
        int y_end = y;
        // verify / redo loop: the state a lane reached at its chunk boundary must be what its left neighbour
        // ended with; the lowest lane that fails runs again from that (exact) state
        int ys = y_b;
        bool run = true, fixed = false;
        for (;;) {
            if (run) {
                int yy = ys, ff = fp_b;
                for (int k = 0; k < nv; ++k) {
                    int v = (int)sm.xf[fm_pidx(base + k)];
                    yy = fm_step<SS>(yy, jb.a1, jb.b0, v, ff);
                    ff = v;
                    sm.fm[fm_pidx(base + k)] = (uint16_t)(int16_t)(SS == 2 ? yy : (yy >> 16));
                }
                y_end = yy;
                fp = ff;
            }
            int prev_end = __shfl_up_sync(0xffffffffu, y_end, 1);
            bool ok = exact || fixed || nv == 0 || y_b == prev_end;
            unsigned bad = __ballot_sync(0xffffffffu, !ok);
            if (!bad) break;
            int const f = __ffs(bad) - 1; // lanes below f are exact
            ys = __shfl_sync(0xffffffffu, y_end, f - 1);
            run = lane == f;
            if (run) fixed = true;
        }
        int const last = (n - 1) / kFmSub;
        int ye = __shfl_sync(0xffffffffu, y_end, last);
        int fe = __shfl_sync(0xffffffffu, fp, last);
        if (lane == 0) {
            sm.fm_state.y = ye;
            sm.fm_state.xf = fe;
        }
    }
    if (lane == 0) {
        sm.fm_state.pos = w0 + n;
        sm.win0 = w0;
        sm.win_n = n;
    }
    __syncwarp();
    if (jb.fm_out) { // stage dump
        for (int i = lane; i < n; i += 32) jb.fm_out[w0 + i] = (int16_t)sm.fm[fm_pidx(i)];
    }
}

// Make a window that holds sample `pos` current: continue the previous window when it ends close in front,
// rebuild the state otherwise (monotone filter).  A filter that is not monotone cannot be rebuilt, but then the
// carrier estimate is not deferred (defer_f1 == 0): f1_evaluate never runs and the walk asks for FM at increasing
// positions only, so the state is never behind w0 and the windows in between are made from it.
// `pos` lies in or in front of the tile being walked; the window ends with that tile (a time slice may end there).
template <int SS>
__device__ R4_NOINLINE void fm_demand(FmJob const &jb, WarpSmem &sm, unsigned long long pos)
{
    constexpr int SPL = 16 / SS;
    unsigned long long const limit = sm.ws.t0 + (unsigned long long)sm.ws.nv_tile;
    unsigned long long w0 = pos / SPL * SPL;
    if (jb.fm_on) {
        unsigned long long const have = sm.fm_state.pos;
        if (jb.monotone && (have > w0 || w0 - have > 2 * kFmWin)) {
            fm_cold<SS>(jb, sm, w0);
        } else {
#ifdef R433B_SIMT_EMU
            assert(have <= w0);
#endif
            while (sm.fm_state.pos + kFmWin <= w0) fm_window<SS>(jb, sm, sm.fm_state.pos, kFmWin); // walk up to it
            w0 = sm.fm_state.pos;
        }
    }
    unsigned long long end = w0 + kFmWin < limit ? w0 + kFmWin : limit;
    fm_window<SS>(jb, sm, w0, (int)(end - w0));
}

// FM of sample `pos` is in sm.fm after this: the current window holds it, or one is made on demand
template <int SS>
__device__ __forceinline__ void fm_cover(FmJob const &jb, WarpSmem &sm, unsigned long long pos)
{
    if (!(sm.win_n > 0 && pos >= sm.win0 && pos < sm.win0 + (unsigned long long)sm.win_n)) fm_demand<SS>(jb, sm, pos);
}

// ---------------------------------------------------- deferred carrier estimate ---------

// src/pulse_detect.c:365 on one sample
__device__ __forceinline__ int f1_step(int g, int f) { return g + f / 64 - g / 64; }

// Evaluate the deferred updates of the carrier estimate: d.ook_f1 holds the exact value in front of the
// first logged sample; the log (entries = runs of consecutive updating samples, relative to the package
// start) is in global memory except for the newest entry.  Returns the exact estimate after the last one.
template <int SS>
__device__ R4_NOINLINE int f1_evaluate(FmJob const &jb, WarpSmem &sm, unsigned const *log, unsigned long long start_abs,
        int g_base, unsigned n_closed, unsigned open_start, unsigned open_count)
{
    int const lane = threadIdx.x & 31;
    // n_closed entries are in global memory, the open one (if any) comes in the arguments
    unsigned const total_entries = n_closed + (open_count ? 1u : 0u);
    if (!total_entries) return g_base;
    auto entry = [&](unsigned i, unsigned &st, unsigned &cnt) {
        if (i < n_closed) {
            st = log[2 * i];
            cnt = log[2 * i + 1];
        } else {
            st = open_start;
            cnt = open_count;
        }
    };
    for (unsigned long long want = kF1Tail;; want *= 4) {
        // the shortest suffix of the log with at least `want` samples
        unsigned j0 = total_entries;
        unsigned long long have = 0;
        while (j0 > 0 && have < want) {
            unsigned st, cnt;
            entry(j0 - 1, st, cnt);
            have += cnt;
            --j0;
        }
        int lo, hi;
        if (j0 == 0) {
            lo = hi = g_base;
        } else { // |g| <= 64 * 512 + 63 always
            lo = -40000;
            hi = 40000;
        }
        for (unsigned j = j0; j < total_entries; ++j) {
            unsigned st, cnt;
            entry(j, st, cnt);
            unsigned long long pos = start_abs + st;
            R4_EMU_ASSERT_POS(pos); // a chunk end folds the log: no entry points in front of the chunk
            while (cnt) {
                fm_cover<SS>(jb, sm, pos);
                unsigned long long wend = sm.win0 + (unsigned long long)sm.win_n;
                unsigned take = wend - pos < cnt ? (unsigned)(wend - pos) : cnt;
                int const i0 = (int)(pos - sm.win0);
                // operands f / 64 of up to 32 samples at a time, lane-parallel into shared memory; the chain then
                // reads four per load
                for (unsigned done = 0; done < take; done += 32) {
                    int const m = take - done < 32 ? (int)(take - done) : 32;
                    __syncwarp();
                    if (lane < m) sm.q[lane] = (int)(int16_t)sm.fm[fm_pidx(i0 + (int)done + lane)] / 64;
                    __syncwarp();
                    int k = 0;
                    if (lo == hi) {
                        for (; k + 4 <= m; k += 4) {
                            int4 const b = *reinterpret_cast<int4 const *>(&sm.q[k]);
                            lo += b.x - lo / 64;
                            lo += b.y - lo / 64;
                            lo += b.z - lo / 64;
                            lo += b.w - lo / 64;
                        }
                        for (; k < m; ++k) lo += sm.q[k] - lo / 64;
                        hi = lo;
                    } else {
                        for (; k < m; ++k) {
                            int const q = sm.q[k];
                            lo += q - lo / 64;
                            hi += q - hi / 64;
                        }
                    }
                }
                pos += take;
                cnt -= take;
            }
        }
        if (lo == hi) return lo;
        // j0 == 0 started from one exact value, so lo == hi there: the loop always ends
    }
}

// ------------------------------------------------------------------ tile hand-over repair ---

// The tile at t0 does not continue the exact filter state `y` (the last AM value in front of it; xp = x[-1] as
// the filter sees it): recompute forward until the values meet the stored ones.  Every lane runs the same
// (warp-uniform) recurrence; lane 0 patches the shared-memory tile, the copy in HBM and the chunk bounds.
template <int SS>
__device__ R4_NOINLINE void am_repair(WarpSmem &sm, uint8_t const *src, unsigned long long t0, int nv_tile, int y, int xp,
        int a1, int b0, unsigned flip, int use_mag, int16_t *am_tile)
{
    int const lane = threadIdx.x & 31;
    uint16_t *am16 = reinterpret_cast<uint16_t *>(sm.am);
    for (int n = 0; n < nv_tile; ++n) {
        int const x = env_at<SS>(src, t0 + (unsigned long long)n, flip, use_mag);
        y = iir16_nowrap(y, a1, b0, x + xp);
        xp = x;
        int const idx = (n >> 6) * (2 * kAmStride) + (n & 63);
        if (y == (int)(int16_t)am16[idx]) break;
        __syncwarp();
        if (lane == 0) {
            am16[idx] = (uint16_t)y;
            am_tile[n] = (int16_t)y;
            int const c = n >> 6;
            if (y < sm.cmin[c]) sm.cmin[c] = y;
            if (y > sm.cmax[c]) sm.cmax[c] = y;
        }
        __syncwarp();
    }
    __syncwarp();
}

// ------------------------------------------------------------- the walk: phases -----------

// The open entry of the deferred carrier-estimate log in registers (warp-uniform); closed entries go to the
// stream's log in global memory.  Entries are runs of consecutive updating samples, relative to the package start.
struct LogRegs {
    unsigned n, start, count;
};
// false: the log is full and has to be folded first (nothing changed)
__device__ __forceinline__ bool log_add(LogRegs &L, unsigned *log, unsigned rel, unsigned cnt, int lane)
{
    if (L.count && L.start + L.count == rel) {
        L.count += cnt;
        return true;
    }
    if (L.count) { // close the open entry
        if (L.n == kLogCap) return false;
        if (lane == 0) {
            log[2 * L.n] = L.start;
            log[2 * L.n + 1] = L.count;
        }
        L.n += 1;
    }
    L.start = rel;
    L.count = cnt;
    return true;
}

// everything logged so far into the exact value ws.d.ook_f1 (state in shared memory)
template <int SS>
__device__ R4_NOINLINE void walk_f1_fold(WarpSmem &sm)
{
    __syncwarp();
    int const g = f1_evaluate<SS>(sm.wc.jb, sm, sm.wc.log, sm.ws.d.start_abs, sm.ws.d.ook_f1, sm.ws.log_n, sm.ws.log_start,
            sm.ws.log_count);
    // the log is not empty, so f1_evaluate synchronised the warp after every lane had read its arguments
    if ((threadIdx.x & 31) == 0) {
        sm.ws.d.ook_f1 = g;
        sm.ws.log_n = 0;
        sm.ws.log_count = 0;
    }
    __syncwarp();
}

// What every entry into pulse_detect_package() does before looking at samples (det_call_boundary), on the state
// in shared memory
__device__ __forceinline__ void walk_call_boundary(WarpSmem &sm)
{
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        if (sm.ws.d.high < sm.wc.lv.min_high) sm.ws.d.high = sm.wc.lv.min_high;
        sm.ws.d.eop_flag = 0;
    }
    __syncwarp();
}

// Hand a finished package over: header + pulse / gap widths into the arenas (state in shared memory)
template <int SS>
__device__ R4_NOINLINE void walk_emit(WarpSmem &sm, int type, unsigned long long pos, bool flush)
{
    int const lane = threadIdx.x & 31;
    __syncwarp();
    if (type == 1 && (sm.ws.log_n || sm.ws.log_count)) walk_f1_fold<SS>(sm); // the carrier estimate of an OOK package is read now
    WalkConst const &wc = sm.wc;
    DetState const d = sm.ws.d;
    unsigned const seq = sm.ws.seq;
    unsigned long long const N = wc.jb.N;
    Trains const tr = wc.tr;
    PackageHeader h = package_header(d, type);
    unsigned cnt = h.num_pulses + 1 < (unsigned)kMaxPulses ? h.num_pulses + 1 : (unsigned)kMaxPulses;
    unsigned idx = 0, off = 0;
    if (lane == 0) {
        idx = atomicAdd(&wc.counters->pkgs, 1u);
        off = atomicAdd(&wc.counters->pool, cnt);
    }
    idx = __shfl_sync(0xffffffffu, idx, 0);
    off = __shfl_sync(0xffffffffu, off, 0);
    bool fits = idx < wc.pkg_cap && (unsigned long long)off + cnt <= wc.pool_cap;
    if (!fits) {
        if (lane == 0) atomicOr(&wc.counters->overflow, 1u);
    } else {
        __syncwarp();
        int const *sp = type == 1 ? tr.ook_pulse : tr.fsk_pulse;
        int const *sg = type == 1 ? tr.ook_gap : tr.fsk_gap;
        for (unsigned i = lane; i < cnt; i += 32) {
            wc.pulse_pool[off + i] = sp[i];
            wc.gap_pool[off + i] = sg[i];
        }
        if (lane == 0) {
            // positions inside the chunk; a chunk is whole blocks, so the block phase is the absolute one and the
            // differences (start_ago: start_abs may lie in front of the chunk, wrapped) are those of the whole file
            unsigned long long blk = flush ? (N + wc.block_samples - 1) / wc.block_samples : pos / wc.block_samples;
            unsigned long long bstart = blk * wc.block_samples;
            unsigned long long blen = flush ? 0 : (N - bstart < wc.block_samples ? N - bstart : wc.block_samples);
            r433b_package k;
            k.stream = wc.stream;
            k.seq = seq;
            k.type = type;
            k.block = (int)(blk + wc.base / wc.block_samples);
            k.offset = h.offset + wc.base;
            k.end_pos = pos + wc.base;
            k.start_ago = flush ? (unsigned)(N - h.start_abs) : (unsigned)(bstart + blen - h.start_abs);
            k.end_ago = flush ? 0u : (unsigned)(blen - (pos - bstart));
            k.num_pulses = h.num_pulses;
            k.pulse_off = off;
            k.pulse_count = cnt;
            k.ook_low_estimate = h.low;
            k.ook_high_estimate = h.high;
            k.fsk_f1_est = h.f1;
            k.fsk_f2_est = h.f2;
            k.first_pair = 0;
            wc.pkgs[idx] = k;
        }
    }
    __syncwarp();
    if (lane == 0) {
        sm.ws.seq = seq + 1;
        sm.ws.log_n = 0;
        sm.ws.log_count = 0;
        sm.ws.pend_type = 0;
    }
    __syncwarp();
}

// AM is signed: it dips to about -350 behind a full-scale sample at a block start (x[-1] narrowed to -32768)
__device__ __forceinline__ int am_tile_at(uint16_t const *am16, int n) { return (int)(int16_t)am16[(n >> 6) * (2 * kAmStride) + (n & 63)]; }

// the IDLE state the noise-floor tracker phases carry in registers
struct IdleRegs {
    int low, high, lead_in;
};

// IDLE over a long stretch of the tile in sm.am from sample n on, lane-parallel: see the comment in the file header
// and below.  While |am - low| < 1024 the tracker is low += (am > low) ? +1 : -1, so low keeps the parity of
// (low0 + samples seen) and two trajectories of equal parity never cross and merge once the data passes between
// them: lane l takes chunk l, starts from a bracket [lo, hi] of the right parity that provably contains the true
// value, pushes both ends through its chunk and hands them to the next lane until the bracket at the end of the
// stretch has collapsed.  Chunks in which a trigger is conceivable (or |am - low| could reach 1024) end the stretch.
// [lo0, hi0] holds the tracker value in front of sample n and has its parity (lo0 == hi0 == d.low when it is known
// exactly; idle_skip starts from a bracket).  `high` must have been derived from `low` already.  Returns the samples
// taken (0: none); d then holds the exact state behind them.
__device__ __forceinline__ int idle_tile(WarpSmem const &sm, IdleRegs &d, int n, int lo0, int hi0, Levels const &lv, int nv_tile)
{
    constexpr int C = kChunk;
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    if (nv_tile - n < 2 * C) return 0;
    int const c0 = n / C;
    int const k0 = lane == c0 ? n - c0 * C : 0;
    int k1 = nv_tile - lane * C;
    k1 = k1 > C ? C : k1;
    bool const in_region = lane >= c0 && k1 > k0;
    // bounds of the chunk's AM values (of the whole chunk for the first, partial one: still bounds)
    int const cmin = in_region ? sm.cmin[lane] : 32767, cmax = in_region ? sm.cmax[lane] : -32768;
    int pmin = cmin, pmax = cmax; // over chunks c0..lane
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t1 = __shfl_up_sync(0xffffffffu, pmin, o);
        int t2 = __shfl_up_sync(0xffffffffu, pmax, o);
        if (lane >= o) {
            pmin = t1 < pmin ? t1 : pmin;
            pmax = t2 > pmax ? t2 : pmax;
        }
    }
    int Lmin = lo0 < pmin - 1 ? lo0 : pmin - 1;
    int Lmax = hi0 > pmax ? hi0 : pmax;
    int const up = lowest_up(Lmin, lv);
    bool const armed = d.lead_in + (nv_tile - n) > kLeadIn;
    bool ok = in_region && !(armed && cmax > up) && (pmax - Lmin < 1024) && (Lmax - pmin < 1024);
    unsigned bad = ~__ballot_sync(0xffffffffu, ok) & (0xffffffffu << c0);
    int const e = bad ? __ffs(bad) - 1 : 32; // chunks c0 .. e-1 form the stretch
    if (e - c0 < 2) return 0;
    int const RLmin = __shfl_sync(0xffffffffu, Lmin, e - 1);
    int const RLmax = __shfl_sync(0xffffffffu, Lmax, e - 1);
    bool const act = lane >= c0 && lane < e;
    int const par = (lo0 + (lane * C + k0 - n)) & 1; // parity of the true value at this lane's start
    // Start bracket.  Over K samples whose values lie in [m, M] the tracker climbs one per sample
    // until it is >= m - 1 and falls one per sample until it is <= M, so from any start in [A, B] it
    // ends in [min(A + K, m - 1), max(B - K, M)].  The chunk to the left has K = 64 samples (the first
    // chunk of the stretch may be partial: then the start bracket and its real length are used).
    int m1 = __shfl_up_sync(0xffffffffu, cmin, 1), M1 = __shfl_up_sync(0xffffffffu, cmax, 1);
    int K1 = __shfl_up_sync(0xffffffffu, k1 - k0, 1);
    int lo, hi;
    if (lane == c0 + 1) {
        lo = lo0 + K1 < m1 - 1 ? lo0 + K1 : m1 - 1;
        hi = hi0 - K1 > M1 ? hi0 - K1 : M1;
    } else {
        lo = RLmin + K1 < m1 - 1 ? RLmin + K1 : m1 - 1;
        hi = RLmax - K1 > M1 ? RLmax - K1 : M1;
    }
    lo = lo < RLmin ? RLmin : lo;
    hi = hi > RLmax ? RLmax : hi;
    lo -= (lo - par) & 1;
    hi += (hi - par) & 1;
    if (lane == c0) {
        lo = lo0;
        hi = hi0;
    }
    int16_t const *chunk = reinterpret_cast<int16_t const *>(am16) + lane * (2 * kAmStride); // signed, as am_tile_at
    int result = 0;
    bool done = false;
#pragma unroll 1
    for (int round = 0; round < 6; ++round) {
        int elo = lo, ehi = hi;
        if (act) {
            if (elo == ehi) {
#pragma unroll 2
                for (int k = k0; k < k1; ++k) elo += (int)chunk[k] > elo ? 1 : -1;
                ehi = elo;
            } else {
#pragma unroll 2
                for (int k = k0; k < k1; ++k) {
                    int a = (int)chunk[k];
                    elo += a > elo ? 1 : -1;
                    ehi += a > ehi ? 1 : -1;
                }
            }
        }
        // the true value lies inside every bracket: a collapsed end bracket is the true value (the first chunk's
        // may never collapse when it starts from a bracket; the last one's decides)
        if (__shfl_sync(0xffffffffu, elo == ehi, e - 1)) {
            result = __shfl_sync(0xffffffffu, elo, e - 1);
            done = true;
            break;
        }
        int nlo = __shfl_up_sync(0xffffffffu, elo, 1);
        int nhi = __shfl_up_sync(0xffffffffu, ehi, 1);
        if (act && lane != c0) {
            lo = nlo;
            hi = nhi;
        }
    }
    if (!done) return 0;
    int const len = (e * C < nv_tile ? e * C : nv_tile) - n;
    d.low = result;
    d.high = derived_high(d.low, lv);
    int li = d.lead_in + len;
    d.lead_in = li > kLeadIn + 1 ? kLeadIn + 1 : li;
    return len;
}

// IDLE from tile sample n on: only the noise-floor tracker moves.  Returns the first sample it could not take
// (a trigger is conceivable there, the tracker leaves its +-1 regime, or `high` has not been re-derived from `low`
// yet after a package): the generic step looks at that one.
__device__ R4_NOINLINE int idle_run(WarpSmem &sm, int n)
{
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    __syncwarp();
    IdleRegs d = {sm.ws.d.low, sm.ws.d.high, sm.ws.d.lead_in};
    Levels const lv = sm.wc.lv;
    int const nv_tile = sm.ws.nv_tile;
    auto am_at = [&](int i) -> int { return am_tile_at(am16, i); };

    // IDLE: only the noise-floor tracker moves (src/pulse_detect.c:325-334).  While
    // |am - low| < 1024 it is low += (am > low) ? +1 : -1; with q = low + j that is
    // q += 2 * (am_j + j > q): two dependent instructions per sample.
    auto idle_fast = [&](int n) -> int {
        int cnt = nv_tile - n < 32 ? nv_tile - n : 32;
        int a = lane < cnt ? am_at(n + lane) : -32768;
        int lmin = d.low - cnt;
        int const up = lowest_up(lmin, lv); // lowest trigger level reachable in this chunk
        bool armed = d.lead_in + cnt - 1 > kLeadIn;
        bool stop = lane < cnt && ((armed && a > up) || (a - lmin >= 1024) || (d.low + cnt - a >= 1024));
        unsigned m = __ballot_sync(0xffffffffu, stop);
        if (m) {
            int first = __ffs(m) - 1;
            cnt = first < cnt ? first : cnt;
        }
        if (cnt == 0) return 0;
        __syncwarp();
        sm.q[lane] = a + lane;
        __syncwarp();
        int q = d.low;
        int j = 0;
#pragma unroll 1
        for (; j + 4 <= cnt; j += 4) {
            int4 const b = *reinterpret_cast<int4 const *>(&sm.q[j]);
            if (b.x > q) q += 2;
            if (b.y > q) q += 2;
            if (b.z > q) q += 2;
            if (b.w > q) q += 2;
        }
#pragma unroll 1
        for (; j < cnt; ++j)
            if (sm.q[j] > q) q += 2;
        d.low = q - cnt;
        d.high = derived_high(d.low, lv);
        int li = d.lead_in + cnt;
        d.lead_in = li > kLeadIn + 1 ? kLeadIn + 1 : li;
        return cnt;
    };


    while (n < nv_tile) {
        if (d.high != derived_high(d.low, lv)) break; // first IDLE sample after a package: not yet re-derived
        int adv = idle_tile(sm, d, n, d.low, d.low, lv, nv_tile);
        if (!adv) adv = idle_fast(n);
        if (!adv) break;
        n += adv;
    }
    __syncwarp();
    if (lane == 0) {
        sm.ws.d.low = d.low;
        sm.ws.d.high = d.high;
        sm.ws.d.lead_in = d.lead_in;
    }
    __syncwarp();
    return n;
}

// Whole IDLE tiles ruled out from k_front's tile summaries, without loading their AM.  Called at the top of the tile
// at t0 in IDLE with `high` derived from `low` (and no package pending); y_am is the exact AM filter state in front
// of t0.  Lane l looks at tile t0 + l of up to 32 tiles per pass.  Tile j is skipped when
//   * it continues tile j - 1: step(last AM of j - 1, x[0] + x[-1]) is its first stored AM.  Lane 0 takes the walk's
//     exact y_am; the others the summary of tile j - 1, which was skipped too and so holds exact AM by induction.
//     k_front's tile is consistent from its first value on, so tile j's stored AM is exact and its summary bounds are
//     real bounds;
//   * the tracker stays in its +-1 regime and no trigger is conceivable anywhere in it: idle_tile's conditions on the
//     whole tile, from the tracker's bracket in front of it.  That is the walk's [lo, hi] on lane 0.  Behind a skipped
//     tile with values in [m, M] it is [m - 1, M] (idle_tile's [min(A + K, m - 1), max(B - K, M)] with K = 2048: the
//     regime conditions keep A, B within 1024 of the values), cut to the parity of `low` in front of t0 (a tile is
//     2048 samples: the parity at every tile start is the same);
//   * it is not the last tile of the launch's range, so a launch always ends on a walked tile (and StreamState holds
//     exact values).
// The prefix of skipped tiles is taken with one ballot.  A block start inside it is a no-op for this state: the call
// boundary clamps `high` to min_high, which a derived `high` already respects, and clears eop_flag, which is zero in
// IDLE (a set flag ends its package at the next sample).
// The exact `low` behind the run is recovered from the last skipped tile's AM by idle_tile's bracket rounds, started
// from the bracket in front of that tile.  Should they not collapse, the run is walked again tile by tile from the
// exact state it started from, up to ws.rewalk_end.  Returns the tile to walk next; ws.skip_y is the AM filter state in
// front of it, ws.d the exact detector state.
#ifndef R4_FORCE_REWALK
#define R4_FORCE_REWALK 0 // tests: 1 = no skipped run is resolved by bracket rounds, every one is walked again
#endif
__device__ R4_NOINLINE unsigned long long idle_skip(WarpSmem &sm, int16_t const *am_stream, ChunkInfo const *chunk_stream,
        unsigned long long t0, unsigned long long sample_end, int y_am, int a1, int b0)
{
    constexpr int T = kTile;
    int const lane = threadIdx.x & 31;
    __syncwarp();
    Levels const lv = sm.wc.lv;
    TileInfo const *const tiles = sm.wc.tiles;
    unsigned long long const range_end = sample_end < sm.wc.jb.N ? sample_end : sm.wc.jb.N; // end of the launch's range
    int const low0 = sm.ws.d.low, lead0 = sm.ws.d.lead_in;
    int const par = low0 & 1;
    int lo = low0, hi = low0, lead = lead0, y = y_am; // in front of tile t
    int plo = 0, phi = 0, plead = 0;                  // in front of the last skipped tile
    unsigned long long t = t0;
#pragma unroll 1
    for (;;) {
        unsigned long long const tl = t + (unsigned long long)lane * T;
        bool const inside = tl + T < range_end;
        TileInfo const ti = inside ? tiles[tl / T] : TileInfo{};
        int const tmin = ti.tmin, tmax = ti.tmax, last = ti.last;
        int const pmin = __shfl_up_sync(0xffffffffu, tmin, 1);
        int const pmax = __shfl_up_sync(0xffffffffu, tmax, 1);
        int const plast = __shfl_up_sync(0xffffffffu, last, 1);
        int blo = pmin - 1, bhi = pmax; // the tracker's bracket in front of this tile
        blo += (blo - par) & 1;
        bhi -= (bhi - par) & 1;
        int yin = plast;
        if (lane == 0) {
            blo = lo;
            bhi = hi;
            yin = y;
        }
        int li = lead + lane * T;
        li = li > kLeadIn + 1 ? kLeadIn + 1 : li;
        int const Lmin = blo < tmin - 1 ? blo : tmin - 1;
        int const Lmax = bhi > tmax ? bhi : tmax;
        bool const armed = li + T > kLeadIn;
        bool const ok = inside && iir16_nowrap(yin, a1, b0, ti.xsum) == (int)ti.first && tmax - Lmin < 1024
                && Lmax - tmin < 1024 && !(armed && tmax > lowest_up(Lmin, lv));
        unsigned const bad = ~__ballot_sync(0xffffffffu, ok);
        int const e = bad ? __ffs(bad) - 1 : 32; // tiles t .. t + e - 1 are skipped
        if (e == 0) break;
        plo = __shfl_sync(0xffffffffu, blo, e - 1);
        phi = __shfl_sync(0xffffffffu, bhi, e - 1);
        plead = __shfl_sync(0xffffffffu, li, e - 1);
        int xlo = tmin - 1, xhi = tmax; // behind this tile
        xlo += (xlo - par) & 1;
        xhi -= (xhi - par) & 1;
        lo = __shfl_sync(0xffffffffu, xlo, e - 1);
        hi = __shfl_sync(0xffffffffu, xhi, e - 1);
        y = __shfl_sync(0xffffffffu, last, e - 1);
        lead = plead + T > kLeadIn + 1 ? kLeadIn + 1 : plead + T;
        t += (unsigned long long)e * T;
        if (e < 32) break;
    }
    if (t != t0) {
        // the exact tracker value behind the run, from the last skipped tile's AM
        unsigned long long const tp = t - T;
        {
            uint4 const *g = reinterpret_cast<uint4 const *>(am_stream + tp + (unsigned long long)(lane * kChunk));
            uint4 v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = g[i];
            ChunkInfo const ci = chunk_stream[tp / kChunk + lane];
            uint32_t *const mine = sm.am + lane * kAmStride;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                mine[4 * i + 0] = v[i].x;
                mine[4 * i + 1] = v[i].y;
                mine[4 * i + 2] = v[i].z;
                mine[4 * i + 3] = v[i].w;
            }
            sm.cmin[lane] = ci.cmin;
            sm.cmax[lane] = ci.cmax;
            __syncwarp();
        }
        IdleRegs d = {plo, 0, plead};
        int const len = R4_FORCE_REWALK ? 0 : idle_tile(sm, d, 0, plo, phi, lv, T);
        __syncwarp();
        if (len == T) {
            if (lane == 0) {
                sm.ws.d.low = d.low;
                sm.ws.d.high = d.high;
                sm.ws.d.lead_in = d.lead_in;
                sm.ws.skip_y = y;
                atomicAdd(&sm.wc.counters->idle_skipped, (unsigned)((t - t0) / T));
            }
            __syncwarp();
            return t;
        }
        // not resolved: the run is walked again from t0 (ws.d still holds the exact state there)
        if (lane == 0) {
            sm.ws.rewalk_end = (unsigned)(t / T);
            atomicAdd(&sm.wc.counters->idle_rewalks, 1u);
        }
    }
    if (lane == 0) sm.ws.skip_y = y_am;
    __syncwarp();
    return t0;
}

// Everything of a package after its first pulse (and the first real gap), in one loop with the hot
// state in registers: src/pulse_detect.c:355-470 without the FSK sub-detector (it is only fed during the
// first pulse) and with the carrier estimate deferred (logged).
//   PULSE: the high-level estimator (:362-363) is a truncating 64-sample moving average -- inherently
//     sequential -- but the pulse only ends on a sample below the threshold its value implies.  One step
//     never lifts `high` above max(high, 64 * (am / 64) + 63), so the largest am of 32 samples bounds
//     every threshold among them from above: samples not below THAT threshold cannot end the pulse.  The
//     recurrence runs over exactly those (operands staged in shared memory, four per load); the first
//     sample that might end the pulse is then tested exactly.
//   GAP_START / GAP: thresholds are frozen; the next event is the first sample above `up` -- a spurious
//     gap if the run is still <= 10 samples, the next pulse otherwise -- or the run length reaching an
//     end-of-package limit (:422-470).  32 samples per ballot.
// Rare turns (spurious pulse, 1200 pulses) are left to det_step() in the generic step: the loop stops in front of the sample.
// Returns the first sample not consumed; a finished package is handed over through pend_type / pend_pos.
__device__ R4_NOINLINE int burst_run(WarpSmem &sm, int n)
{
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    __syncwarp();
    struct {
        int st, run, high, low, longest, last_pulse;
        unsigned ook_n, ook_hw;
        unsigned long long start_abs;
    } d = {sm.ws.d.st, sm.ws.d.run, sm.ws.d.high, sm.ws.d.low, sm.ws.d.longest, sm.ws.d.last_pulse,
           sm.ws.d.ook_n, sm.ws.d.ook_hw, sm.ws.d.start_abs};
    LogRegs L = {sm.ws.log_n, sm.ws.log_start, sm.ws.log_count};
    Levels const lv = sm.wc.lv;
    Trains const tr = sm.wc.tr;
    unsigned *const log = sm.wc.log;
    int const per_ms = sm.wc.per_ms;
    int const nv_tile = sm.ws.nv_tile;
    unsigned long long const t0 = sm.ws.t0;
    int pend_type = 0;
    unsigned long long pend_pos = 0;
    auto am_at = [&](int i) -> int { return am_tile_at(am16, i); };
    int st = d.st, run = d.run, h = d.high;
    int const low = d.low, minh = lv.min_high;
#pragma unroll 1
    while (n < nv_tile) {
        if (st == kPulse) {
            if (d.ook_n == 0) break; // a first pulse feeds the FSK sub-detector: not here
            unsigned const rel = (unsigned)(t0 + (unsigned long long)n - d.start_abs);
            // a full log is folded by the generic step first (nothing has been touched yet)
            if (L.count && L.start + L.count != rel && L.n == kLogCap) break;
            int cnt = nv_tile - n < 32 ? nv_tile - n : 32;
            int const a = lane < cnt ? am_at(n + lane) : 32767;
            // am / 64 as :362 computes it: AM dips below zero behind a full-scale sample at a block start, and such a
            // sample is taken here when `down` is negative (`low` below zero, min_level far below its default)
            int const aq = a / 64;
            int const top = __reduce_max_sync(0xffffffffu, lane < cnt ? aq : 0); // one REDUX each
            int hmax = 64 * top + 63;
            hmax = h > hmax ? h : hmax;
            int const dn = det_thresholds(low, hmax, lv).down;
            unsigned const m = __ballot_sync(0xffffffffu, lane < cnt && a < dn);
            if (m) cnt = __ffs(m) - 1;
            if (cnt) {
                __syncwarp();
                sm.q[lane] = aq;
                __syncwarp();
                // h >= min_high >= 0 here, so h / 64 == h >> 6.  Eight steps per trip, the loops kept rolled: seven
                // warps per scheduler share an instruction cache of a few hundred instructions.
                // With dn >= 0 every sample taken has q >= 0, so one step takes at most h >> 6 off, and less from a
                // lower h: after k steps h is still >= h0 - k (h0 >> 6).  If that stays >= min_high over the whole
                // stretch the clamp of :363 cannot act and is left out of the dependency chain.
                int4 const *qp = reinterpret_cast<int4 const *>(sm.q);
                int trips = cnt >> 3;
#define R4_STEP(q) h += (q) - (int)((unsigned)h >> 6)
#define R4_STEP_CLAMPED(q) h = max(h + (q) - (int)((unsigned)h >> 6), minh)
                if (dn >= 0 && h - cnt * (int)((unsigned)h >> 6) >= minh) {
#pragma unroll 1
                    for (; trips > 0; --trips, qp += 2) {
                        int4 const b = qp[0], c = qp[1];
                        R4_STEP(b.x); R4_STEP(b.y); R4_STEP(b.z); R4_STEP(b.w);
                        R4_STEP(c.x); R4_STEP(c.y); R4_STEP(c.z); R4_STEP(c.w);
                    }
                } else {
#pragma unroll 1
                    for (; trips > 0; --trips, qp += 2) {
                        int4 const b = qp[0], c = qp[1];
                        R4_STEP_CLAMPED(b.x); R4_STEP_CLAMPED(b.y); R4_STEP_CLAMPED(b.z); R4_STEP_CLAMPED(b.w);
                        R4_STEP_CLAMPED(c.x); R4_STEP_CLAMPED(c.y); R4_STEP_CLAMPED(c.z); R4_STEP_CLAMPED(c.w);
                    }
                }
#undef R4_STEP
#undef R4_STEP_CLAMPED
                {
                    int const *qs = reinterpret_cast<int const *>(qp);
#pragma unroll 1
                    for (int r = cnt & 7; r > 0; --r, ++qs) h = max(h + *qs - (int)((unsigned)h >> 6), minh);
                }
                log_add(L, log, rel, (unsigned)cnt, lane);
                run += cnt;
                n += cnt;
            }
            if (m) { // the sample at n might end the pulse: the exact test of :355
                int const aj = __shfl_sync(0xffffffffu, a, cnt);
                if (aj < det_thresholds(low, h, lv).down) {
                    if (run + 1 < kMinPulseSamples) break; // spurious pulse (:341-350)
                    run += 1;
                    put(tr.ook_pulse, d.ook_hw, d.ook_n, run);
                    d.last_pulse = run;
                    if (run > d.longest) d.longest = run;
                    run = 0;
                    st = kGapStart;
                } else {
                    h += aj / 64 - (int)((unsigned)h >> 6);
                    h = h < minh ? minh : h;
                    log_add(L, log, (unsigned)(t0 + (unsigned long long)n - d.start_abs), 1u, lane);
                    run += 1;
                }
                n += 1;
            }
            continue;
        }
        // GAP_START (run <= 9 so far) or GAP
        int const cnt = nv_tile - n;
        int const up = det_thresholds(low, h, lv).up;
        // min(max(10 * longest, 10 * per_ms), 100 * per_ms) in 32 bits: a pulse of 10 * per_ms samples or more makes
        // the first limit reach the second, so `longest` can be capped there (per_ms <= 2^31 / 1000: no overflow)
        int const lim_b = 100 * per_ms;
        int const lcap = d.longest < 10 * per_ms ? d.longest : 10 * per_ms;
        int const lim_a = lcap > per_ms ? 10 * lcap : 10 * per_ms;
        int const rstar = (lim_a < lim_b ? lim_a : lim_b) + 1; // first run length that ends the package
        int je = rstar - run - 1;                               // ... reached at this sample of the scan
        // the limits are only looked at in GAP, i.e. from the sample after the one that brought the run to 10
        int const first_gap = st == kGapStart ? kMinPulseSamples - run : 0;
        if (je < first_gap) je = first_gap;
        int const horizon = je < cnt ? je + 1 : cnt; // samples that matter
        int ja = 0x7fffffff;
#pragma unroll 1
        for (int base = 0; base < horizon; base += 32) {
            int const a = base + lane < cnt ? am_at(n + base + lane) : -32768;
            unsigned const m = __ballot_sync(0xffffffffu, a > up);
            if (m) {
                ja = base + __ffs(m) - 1;
                break;
            }
        }
        if (ja < cnt && ja <= je) {
            if (st == kGapStart && run + ja + 1 <= kMinPulseSamples) { // spurious gap (:379-385)
                run += ja + 1 + d.last_pulse;
                st = kPulse;
                n += ja + 1;
                continue;
            }
            if (d.ook_n + 1 >= (unsigned)kMaxPulses) { // the 1200th pulse ends the package (:429-441): det_step()
                run += ja;
                n += ja;
                st = run >= kMinPulseSamples ? kGap : kGapStart;
                break;
            }
            run += ja + 1; // a new pulse starts (:422-428)
            put(tr.ook_gap, d.ook_hw, d.ook_n, run);
            d.ook_n += 1;
            run = 0;
            st = kPulse;
            n += ja + 1;
            continue;
        }
        if (je < cnt) { // end of package by gap length (:443-469)
            run += je + 1;
            put(tr.ook_gap, d.ook_hw, d.ook_n, run);
            d.ook_n += 1;
            st = kIdle;
            pend_type = 1;
            n += je; // that sample is looked at again in IDLE
            pend_pos = t0 + (unsigned long long)n;
            break;
        }
        run += cnt;
        if (run >= kMinPulseSamples) st = kGap;
        n += cnt;
    }
    d.st = st;
    d.run = run;
    d.high = h;

    __syncwarp();
    if (lane == 0) {
        sm.ws.d.st = d.st;
        sm.ws.d.run = d.run;
        sm.ws.d.high = d.high;
        sm.ws.d.longest = d.longest;
        sm.ws.d.last_pulse = d.last_pulse;
        sm.ws.d.ook_n = d.ook_n;
        sm.ws.d.ook_hw = d.ook_hw;
        sm.ws.log_n = L.n;
        sm.ws.log_start = L.start;
        sm.ws.log_count = L.count;
        if (pend_type) {
            sm.ws.pend_type = pend_type;
            sm.ws.pend_pos = pend_pos;
        }
    }
    __syncwarp();
    return n;
}

// The FIRST pulse of a package, from tile sample n on (src/pulse_detect.c:355-374 with ook_n == 0): the high-level
// estimator, the carrier estimate (not yet deferred) and the FSK sub-detector are fed sample by sample -- an FSK
// transmission is one long OOK "pulse", so this is the hot loop of FSK captures.  The same bound as in
// burst_run() tells which samples cannot end the pulse; the first one that might is left to the generic step.
// Reads FM: windows are made current as the walk reaches them.  Returns the first sample not consumed.
template <int SS>
__device__ R4_NOINLINE int first_run(WarpSmem &sm, int n)
{
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    __syncwarp();
    struct {
        int high, run, ook_f1;
        unsigned fsk_n, fsk_hw;
        unsigned long long fsk_offset;
        unsigned fk_len;
        int fk_st, fk_f1, fk_f2, fk_vmax, fk_vmin, fk_skip;
    } d = {sm.ws.d.high, sm.ws.d.run, sm.ws.d.ook_f1, sm.ws.d.fsk_n, sm.ws.d.fsk_hw, sm.ws.d.fsk_offset, sm.ws.d.fk_len,
           sm.ws.d.fk_st, sm.ws.d.fk_f1, sm.ws.d.fk_f2, sm.ws.d.fk_vmax, sm.ws.d.fk_vmin, sm.ws.d.fk_skip};
    int const low = sm.ws.d.low;
    Levels const lv = sm.wc.lv;
    Trains const tr = sm.wc.tr;
    int const fpdm = sm.wc.fpdm, minh = lv.min_high;
    int const nv_tile = sm.ws.nv_tile;
    unsigned long long const t0 = sm.ws.t0;
    WarpCtx cx;
    cx.lane = lane;
    cx.nlanes = 32;
#pragma unroll 1
    while (n < nv_tile) {
        unsigned long long const pos = t0 + (unsigned long long)n;
        fm_cover<SS>(sm.wc.jb, sm, pos);
        int cnt = nv_tile - n < 32 ? nv_tile - n : 32;
        int const in_win = (int)(sm.win0 + (unsigned long long)sm.win_n - pos);
        cnt = cnt < in_win ? cnt : in_win;
        int const a = lane < cnt ? am_tile_at(am16, n + lane) : 32767;
        int const f = lane < cnt ? (int)(int16_t)sm.fm[fm_pidx((int)(pos - sm.win0) + lane)] : 0;
        int const aq = a / 64; // as in burst_run
        int const top = __reduce_max_sync(0xffffffffu, lane < cnt ? aq : 0);
        int hmax = 64 * top + 63;
        hmax = d.high > hmax ? d.high : hmax;
        unsigned const m = __ballot_sync(0xffffffffu, lane < cnt && a < det_thresholds(low, hmax, lv).down);
        if (m) cnt = __ffs(m) - 1;
        if (cnt) {
            __syncwarp();
            sm.q[lane] = (aq << 16) | (f & 0xffff); // one word per sample: am / 64 above, FM below
            __syncwarp();
#pragma unroll 1
            for (int j = 0; j < cnt; ++j) {
                int const w = sm.q[j];
                int const fj = (int)(int16_t)(w & 0xffff);
                d.high = max(d.high + (w >> 16) - (int)((unsigned)d.high >> 6), minh);
                d.ook_f1 += fj / 64 - d.ook_f1 / 64;
                if (fpdm == 0)
                    fsk_classic(d, tr, fj, cx);
                else
                    fsk_minmax(d, tr, fj, cx);
            }
            d.run += cnt;
            n += cnt;
        }
        if (m) break; // this sample might end the pulse: the generic step tests it exactly
    }
    __syncwarp();
    if (lane == 0) {
        sm.ws.d.high = d.high;
        sm.ws.d.run = d.run;
        sm.ws.d.ook_f1 = d.ook_f1;
        sm.ws.d.fsk_n = d.fsk_n;
        sm.ws.d.fsk_hw = d.fsk_hw;
        sm.ws.d.fsk_offset = d.fsk_offset;
        sm.ws.d.fk_len = d.fk_len;
        sm.ws.d.fk_st = d.fk_st;
        sm.ws.d.fk_f1 = d.fk_f1;
        sm.ws.d.fk_f2 = d.fk_f2;
        sm.ws.d.fk_vmax = d.fk_vmax;
        sm.ws.d.fk_vmin = d.fk_vmin;
        sm.ws.d.fk_skip = d.fk_skip;
    }
    __syncwarp();
    return n;
}

// Everything else, one sample (or one stretch of a first pulse) at a time: package starts, first pulses with
// the FSK sub-detector (they read FM), spurious pulses, the 1200th pulse, filters that rule the deferred
// estimate out.  Always makes progress: it consumes at least one sample or hands a package over (ws.pend_type).
template <int SS>
__device__ R4_NOINLINE int generic_step(WarpSmem &sm, int n)
{
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    __syncwarp();
    DetState d = sm.ws.d;
    LogRegs L = {sm.ws.log_n, sm.ws.log_start, sm.ws.log_count};
    Levels const lv = sm.wc.lv;
    Trains const tr = sm.wc.tr;
    unsigned *const log = sm.wc.log;
    int const per_ms = sm.wc.per_ms, fpdm = sm.wc.fpdm;
    bool const defer_f1 = sm.wc.defer_f1 != 0;
    unsigned long long const t0 = sm.ws.t0;
    WarpCtx cx;
    cx.lane = lane;
    cx.nlanes = 32;
    auto am_at = [&](int i) -> int { return am_tile_at(am16, i); };
    auto store = [&]() {
        __syncwarp();
        if (lane == 0) {
            sm.ws.d = d;
            sm.ws.log_n = L.n;
            sm.ws.log_start = L.start;
            sm.ws.log_count = L.count;
        }
        __syncwarp();
    };
    auto log_append = [&](unsigned long long pos, unsigned cnt) {
        unsigned const rel = (unsigned)(pos - d.start_abs);
        if (log_add(L, log, rel, cnt, lane)) return;
        store(); // the log is full: fold it into the exact value first
        walk_f1_fold<SS>(sm);
        d.ook_f1 = sm.ws.d.ook_f1;
        L.n = L.count = 0;
        log_add(L, log, rel, cnt, lane);
    };
    auto fm_at = [&](int i) -> int { return (int)(int16_t)sm.fm[fm_pidx((int)(t0 + (unsigned long long)i - sm.win0))]; };

    // inside a first pulse (and its GAP_START) the FSK sub-detector and the undeferred estimate read FM
    bool const first = d.ook_n == 0 && (d.st == kPulse || d.st == kGapStart);
    bool const wants_fm = first || (d.st == kPulse && !defer_f1);
    if (wants_fm) fm_cover<SS>(sm.wc.jb, sm, t0 + (unsigned long long)n);
    int adv = 0;
    {
        // every lane runs the (warp-uniform) step and writes the same train entries: keep the lanes
        // together so that no lane reads an entry another lane has already overwritten for a later sample
        __syncwarp();
        int const r = det_step<kStepAll>(d, lv, tr, am_at(n), wants_fm ? fm_at(n) : 0, t0 + n, per_ms, fpdm, cx, defer_f1);
        if (r & kStepF1Deferred) log_append(t0 + (unsigned long long)n, 1u);
        if (r & 3) {
            // the same sample is examined again, now in IDLE
            __syncwarp();
            if (lane == 0) {
                sm.ws.pend_type = r & 3;
                sm.ws.pend_pos = t0 + (unsigned long long)n;
            }
        } else {
            if (d.st == kPulse && d.run == 0 && d.ook_n == 0) L.n = L.count = 0; // a package has just begun
            adv = 1;
        }
    }
    store();
    return n + adv;
}

// The end of a chunk of a file that goes on in the next chained batch (the launch that reaches it has walked its last
// tile: idle_skip never skips the last tile of a range).  Nothing the next chunk reads may lie in front of it: the
// deferred carrier-estimate log is folded into its exact value, the FM filter state is made exact at the chunk end (a
// monotone filter by range collapse, which reaches back no further than the state known in this chunk; any other
// forward from the last exact state), and the chunk's last IQ sample is kept.  Positions are rebased to the next
// chunk's sample 0.  `ss` receives what the next chunk starts from.
template <int SS>
__device__ R4_NOINLINE void chunk_end(WarpSmem &sm, StreamState *ss)
{
    int const lane = threadIdx.x & 31;
    __syncwarp();
    FmJob const &jb = sm.wc.jb;
    unsigned long long const N = jb.N;
    if (sm.ws.log_n || sm.ws.log_count) {
        walk_f1_fold<SS>(sm);
        if (lane == 0) atomicAdd(&sm.wc.counters->chain_folds, 1u);
    }
    if (jb.fm_on && sm.fm_state.pos != N) {
        if (jb.monotone) {
            fm_cold<SS>(jb, sm, N);
        } else {
            while (sm.fm_state.pos < N) {
                unsigned long long const w0 = sm.fm_state.pos;
                fm_window<SS>(jb, sm, w0, N - w0 < (unsigned long long)kFmWin ? (int)(N - w0) : kFmWin);
            }
        }
        if (lane == 0) atomicAdd(&sm.wc.counters->chain_fm_rebuilds, 1u);
    }
    int ci, cq;
    iq_at<SS>(jb.src, N - 1, jb.flip, ci, cq);
    __syncwarp();
    if (lane == 0) {
        if (!jb.fm_on) sm.fm_state = FmState{N, 0, 0}; // unused: "FM" is the raw envelope
        sm.fm_state.pos -= N;
        sm.ws.d.start_abs -= N;
        sm.ws.d.fsk_offset -= N;
        ss->fm_start = sm.fm_state;
        ss->iq_i = ci;
        ss->iq_q = cq;
    }
    __syncwarp();
}

// --------------------------------------------------------------------------- kernel ------

template <int SS>
__global__ void __launch_bounds__(kDetectWarps * 32, kDetectCtasPerSm) k_detect(DetectParams p)
{
    constexpr int C = kChunk;
    constexpr int T = kTile;
    R4_DYN_SMEM(uint32_t, smem_raw);

    int const warp = threadIdx.x >> 5;
    int const lane = threadIdx.x & 31;
    unsigned const s = p.stream0 + blockIdx.x * kDetectWarps + warp;
    if (s >= p.stream_end) return;

    WarpSmem &sm = reinterpret_cast<WarpSmem *>(smem_raw)[warp];
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);

    unsigned long long const byte0 = p.offsets[s];
    unsigned long long const N = (p.lengths ? p.lengths[s] : p.offsets[s + 1] - byte0) / SS;
    uint8_t const *const src = p.data + byte0;
    int16_t *const am_stream = p.am + p.am_offsets[s];
    ChunkInfo const *const chunk_stream = p.chunks + p.am_offsets[s] / kChunk;
    // the deferred carrier estimate re-makes FM for logged samples later, out of order: needs the state rebuild
    bool const defer_f1 = !p.enable_fm || p.wrap_free != 0;

    int y_am = 0; // the last AM value of the previous tile: the AM filter state (reset_sdr_flow(): zero)
    int flushed = 0;
    // a stream that continues a file (chained batch) loads its state in the batch's first launch too
    bool const fresh = p.first_chunk && !(p.cont && p.cont[s]);
    if (lane == 0) {
        WalkConst &wc = sm.wc;
        wc.jb.src = src;
        wc.jb.N = N;
        wc.jb.flip = p.flip;
        wc.jb.a1 = p.fm_a1;
        wc.jb.b0 = p.fm_b0;
        wc.jb.fm_on = p.enable_fm;
        wc.jb.use_mag = p.use_mag;
        wc.jb.monotone = p.wrap_free;
        wc.jb.fm_out = nullptr;
        wc.tr.ook_pulse = p.train_scratch + (size_t)s * kTrainInts;
        wc.tr.ook_gap = wc.tr.ook_pulse + kMaxPulses;
        wc.tr.fsk_pulse = wc.tr.ook_gap + kMaxPulses;
        wc.tr.fsk_gap = wc.tr.fsk_pulse + kMaxPulses;
        wc.log = p.log_scratch + (size_t)s * kLogCap * 2;
        wc.lv = p.lv;
        wc.per_ms = (int)(p.rate / 1000);
        wc.fpdm = p.fpdm;
        wc.defer_f1 = defer_f1;
        wc.stream = s;
        wc.block_samples = p.block_samples;
        wc.base = p.base ? p.base[s] : 0;
        wc.pkgs = p.pkgs;
        wc.pulse_pool = p.pulse_pool;
        wc.gap_pool = p.gap_pool;
        wc.pkg_cap = p.pkg_cap;
        wc.pool_cap = p.pool_cap;
        wc.counters = p.counters;
        wc.tiles = p.tile_info ? p.tile_info + p.am_offsets[s] / kTile : nullptr;
        WalkState &ws = sm.ws;
        ws.pend_type = 0;
        ws.pend_pos = 0;
        ws.t0 = 0;
        ws.nv_tile = 0;
        ws.skip_y = 0;
        ws.rewalk_end = 0;
        if (fresh) {
            det_reset(ws.d);
            ws.d.ook_hw = ws.d.fsk_hw = kMaxPulses; // scratch is not assumed to be zero: first package clears it
            ws.log_n = ws.log_start = ws.log_count = 0;
            ws.seq = 0;
            sm.fm_state = FmState{0, 0, 0};
            wc.jb.start = FmState{0, 0, 0};
            wc.jb.pri0 = wc.jb.prq0 = 0;
            if (p.state) {
                p.state[s].fm_start = wc.jb.start;
                p.state[s].iq_i = p.state[s].iq_q = 0;
            }
        } else {
            StreamState const &ss = p.state[s];
            ws.d = ss.d;
            ws.seq = ss.seq;
            ws.log_n = ss.log_n;
            ws.log_start = ss.last_start;
            ws.log_count = ss.last_count;
            sm.fm_state = ss.fm_state;
            wc.jb.start = ss.fm_start;
            wc.jb.pri0 = ss.iq_i;
            wc.jb.prq0 = ss.iq_q;
        }
        sm.win0 = 0;
        sm.win_n = 0;
    }
    if (!fresh) y_am = p.state[s].y_am;
    if (!p.first_chunk) flushed = p.state[s].flushed;
    __syncwarp();

    int const a1 = p.lpf_a1, b0 = p.lpf_b0;

    for (unsigned long long t0 = p.sample_begin; t0 < p.sample_end && t0 < N; t0 += T) {
        if (sm.wc.tiles && sm.ws.d.st == kIdle && !sm.ws.pend_type && !sm.ws.d.eop_flag && t0 / T >= sm.ws.rewalk_end) {
            if (sm.ws.d.high == derived_high(sm.ws.d.low, p.lv)) {
                t0 = idle_skip(sm, am_stream, chunk_stream, t0, p.sample_end, y_am, a1, b0);
                y_am = sm.ws.skip_y;
            }
        }
        unsigned long long const remain = N - t0;
        int const nv_tile = remain < (unsigned long long)T ? (int)remain : T;

        // ---- AM tile from HBM ---------------------------------------------------------------------
        // every load of the tile is issued before anything waits for one: the AM line of the lane's chunk, the
        // chunk bounds, the two IQ samples of the hand-over check; the next tile is pulled into L2 meanwhile
        {
            uint4 const *g = reinterpret_cast<uint4 const *>(am_stream + t0 + (unsigned long long)(lane * C));
            uint4 v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = g[i];
            ChunkInfo const ci = chunk_stream[t0 / C + lane];
            // the first tile of a stream starts from the reset state in k_front, the first of a continued chunk from the
            // carried state (exact as well, but checked: it is the tile a spoiled guess of the tests lands on)
            bool const handover = t0 != 0 || (p.cont && p.cont[s]); // t0 == 0: read here, not kept live across the walk
            int x0 = 0, xm = 0;
            if (handover) {
                x0 = env_at<SS>(src, t0, p.flip, p.use_mag);
                xm = t0 != 0 ? env_at<SS>(src, t0 - 1, p.flip, p.use_mag) : env_iq<SS>(sm.wc.jb.pri0, sm.wc.jb.prq0, p.use_mag);
            }
#ifndef R433B_SIMT_EMU
            if (t0 + T < N) {
                asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<char const *>(g) + T * sizeof(int16_t)));
                if (lane == 0) {
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(chunk_stream + (t0 + T) / C));
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(src + (t0 + T) * SS));
                }
            }
#endif
            uint32_t *const mine = sm.am + lane * kAmStride;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                mine[4 * i + 0] = v[i].x;
                mine[4 * i + 1] = v[i].y;
                mine[4 * i + 2] = v[i].z;
                mine[4 * i + 3] = v[i].w;
            }
            bool const has = lane * C < nv_tile;
            sm.cmin[lane] = has ? (int)ci.cmin : 32767;
            sm.cmax[lane] = has ? (int)ci.cmax : 0;
            if (lane == 0) {
                sm.ws.t0 = t0;
                sm.ws.nv_tile = nv_tile;
            }
            __syncwarp();
            // hand-over check (see the file header)
            if (handover) {
                // the reference keeps x[-1] as int16 across block calls (src/baseband.c:167)
                if (t0 % p.block_samples == 0) xm = (int)(int16_t)xm;
                int const expect = iir16_nowrap(y_am, a1, b0, x0 + xm);
                if (expect != (int)(int16_t)am16[0]) {
                    am_repair<SS>(sm, src, t0, nv_tile, y_am, xm, a1, b0, p.flip, p.use_mag, am_stream + t0);
                    if (lane == 0) atomicAdd(&p.counters->front_repairs, 1u);
                }
            }
        }
        y_am = am_tile_at(am16, nv_tile - 1);

        // ---- package detector over the tile (warp-uniform), phase by phase ------------------------
        if (t0 % p.block_samples == 0) walk_call_boundary(sm);
        for (int n = 0; n < nv_tile;) {
            int const st = sm.ws.d.st;
            int m = n;
            if (st == kIdle)
                m = idle_run(sm, n);
            // burst_run leaves out the FSK hand-over of GAP_START (:387): the first pulse's GAP_START may feed the FSK
            // sub-detector its 17th pulse on the sample it moves to GAP, and then the next GAP_START ends the package
            else if (defer_f1 && !sm.ws.d.eop_flag && (sm.ws.d.ook_n != 0 || st == kGap) && sm.ws.d.fsk_n <= (unsigned)kMinPulses)
                m = burst_run(sm, n);
            else if (st == kPulse && sm.ws.d.ook_n == 0)
                m = first_run<SS>(sm, n);
            if (m == n && !sm.ws.pend_type) m = generic_step<SS>(sm, n);
            n = m;
            if (sm.ws.pend_type) { // a package to hand over; the sample at n is looked at again
                walk_emit<SS>(sm, sm.ws.pend_type, sm.ws.pend_pos, false);
                walk_call_boundary(sm);
            }
        }
        __syncwarp();
    }

    // flush_sdr_flow(): len == 0 call(s) at the end of the file, in the launch that reaches it; the end of a chunk of a
    // file that goes on hands its state to the next chunk instead
    if (N <= p.sample_end && !flushed && p.last && !p.last[s]) {
        if (N) chunk_end<SS>(sm, p.state + s);
        flushed = 1;
    }
    if (N <= p.sample_end && !flushed) {
        for (;;) {
            __syncwarp();
            DetState d = sm.ws.d;
            int const ev = det_flush(d, sm.wc.tr, p.fpdm);
            __syncwarp();
            if (lane == 0) sm.ws.d = d;
            __syncwarp();
            if (!ev) break;
            walk_emit<SS>(sm, ev, N, true);
        }
        flushed = 1;
    }
    __syncwarp();
    if (lane == 0 && p.state) {
        StreamState &ss = p.state[s];
        ss.d = sm.ws.d;
        ss.y_am = y_am;
        ss.fm_state = sm.fm_state;
        ss.log_n = sm.ws.log_n;
        ss.last_start = sm.ws.log_start;
        ss.last_count = sm.ws.log_count;
        ss.seq = sm.ws.seq;
        ss.flushed = flushed;
    }

    // ---- stage dump: FM (the raw envelope with FM off) of every sample, after the walk and apart from it ----------
    // From the state in front of sample 0 over [0, N): the host gives a batch with stage arrays one launch over whole
    // streams (chunks).
    if (p.fm_out) {
        if (lane == 0) {
            sm.wc.jb.fm_out = p.fm_out + byte0 / SS; // the walk is over: its job can take the dump
            sm.fm_state = sm.wc.jb.start;
        }
        __syncwarp();
        for (unsigned long long w0 = 0; w0 < N; w0 += kFmWin)
            fm_window<SS>(sm.wc.jb, sm, w0, N - w0 < (unsigned long long)kFmWin ? (int)(N - w0) : kFmWin);
    }
}

} // namespace r433b
