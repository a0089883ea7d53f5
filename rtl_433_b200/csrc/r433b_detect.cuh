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
//
//  2. The package detector (src/pulse_detect.c:199-483) walks the tile warp-uniformly with ballot scans for
//     the states whose thresholds are frozen (IDLE stretches by bracket rounds, GAP, GAP_START) and a
//     sequential but lean recurrence for the high-level estimator of PULSE.
//
//  3. FM (src/baseband.c:181-366) is only READ in two places: by the FSK sub-detector during the first
//     pulse of a package, and by the carrier estimate `fsk_f1_est`, which is reported when a package ends.
//     Neither needs FM for every sample:
//       * FM WINDOWS of 256 samples are made on demand (discriminator lane-parallel from the IQ bytes,
//         low-pass by sub-chunks with the same start-from-a-guess / verify / redo scheme).  The filter state
//         in front of a window that does not continue the previous one is rebuilt RIGOROUSLY: both ends of
//         the whole state range are pushed through the samples in front of the window until they meet
//         (monotone filter: the host proves a1, b0 >= 0, a1 + 2 b0 <= unity; otherwise FM is made for
//         every window of every tile).
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

#ifndef R4_REC
#define R4_REC 2 // recurrence loop of burst_run: 0 always clamped, 1 clamp decided per 8 steps, 2 per stretch
#endif
namespace r433b {

constexpr int kTrainInts = 4 * kMaxPulses; // per-stream scratch: ook pulse/gap, fsk pulse/gap
constexpr int kDetectWarps = 4;            // warps (streams) per CTA
constexpr int kDetectCtasPerSm = 8;        // 32 warps per SM (64 registers): 4096 streams are co-resident on 132 SMs

constexpr int kAmStride = kChunk / 2 + 1;  // words between lane chunks of the 16-bit AM tile (odd: conflict-free)
constexpr int kAmWords = 32 * kAmStride;
constexpr int kFmWin = 256;                // FM window
constexpr int kFmSub = kFmWin / 32;        // samples per lane of a window
constexpr int kFmPadded = kFmWin + kFmWin / kFmSub; // padded index space: i + i / kFmSub
constexpr int kWarmFm = 48;                // warm-up samples of the FM trajectories
constexpr int kFmWindowsPerTile = kTile / kFmWin;
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
    unsigned flip;
    long long a1, b0;
    int fm_on;                 // 0: "FM" is the raw envelope (buf.fm aliases buf.temp when nothing asks for FM)
    int use_mag;
    int monotone;              // the state rebuild by range collapse is valid
    int16_t *fm_out;           // stage dump (absolute index = stream base + sample) or nullptr
};

// Warp-uniform state of the walk.  It lives in shared memory BETWEEN the phases of the walk (idle_run, burst_run,
// generic_step, walk_emit: separate functions, each with the registers and the instruction footprint of its own
// loop); a phase loads what it needs into registers, every lane computes the same values, lane 0 stores them back.
struct WalkState {
    DetState d;
    unsigned log_n, log_start, log_count; // deferred carrier-estimate log: closed entries (global memory), the open entry
    unsigned seq;
    int pend_type;               // a finished package to hand over (1 OOK, 2 FSK) ...
    unsigned long long pend_pos; // ... returned at this stream position
    unsigned long long t0;       // the tile being walked
    int nv_tile;
};

// Per-stream constants of the walk (written once by lane 0)
struct WalkConst {
    FmJob jb;
    Trains tr;
    unsigned *log;
    Levels lv;
    int per_ms, fpdm, lazy_fm, defer_f1;
    unsigned stream, block_samples;
    r433b_package *pkgs;
    int *pulse_pool, *gap_pool;
    unsigned pkg_cap, pool_cap;
    unsigned *counters;
};

// Shared memory of one warp
struct alignas(16) WarpSmem {
    uint32_t am[kAmWords];       // AM tile, 16 bits per sample: sample n at u16 (n / 64) * 66 + n % 64
    uint32_t xf[kFmPadded];      // discriminator outputs of the current FM window (padded index)
    uint16_t fm[kFmPadded];      // FM (or the raw-envelope alias) of the current window
    int q[32];                   // chain operands of one 32-sample step
    int cmin[32], cmax[32];      // per lane chunk: bounds of its AM values
    // FM bookkeeping (warp-uniform; written by lane 0)
    unsigned long long fm_pos;   // (fm_y, fm_xf) is the exact filter state after sample fm_pos - 1
    int fm_y, fm_xf;
    unsigned long long win0;     // the window holds FM of [win0, win0 + win_n)
    int win_n;
    int tile_state_y[kFmWindowsPerTile], tile_state_xf[kFmWindowsPerTile]; // eager mode: state in front of each window
    unsigned long long tile_end_pos; // eager mode: the contiguous filter state at the end of the tile pass
    int tile_end_y, tile_end_xf;
    WalkState ws;
    WalkConst wc;
};

// Everything one stream carries from one launch to the next when a batch is processed in time slices.
struct StreamState {
    DetState d;
    int y_am;
    unsigned long long fm_pos;
    int fm_y, fm_xf;
    unsigned log_n, last_start, last_count;
    unsigned seq;
    int flushed;
};

struct DetectParams {
    uint8_t const *data;
    unsigned long long const *offsets; // bytes, n_streams + 1
    unsigned long long const *lengths; // optional: bytes of stream i actually used
    unsigned long long const *am_offsets; // first sample of stream i in `am` (k_front's output)
    unsigned n_streams;
    unsigned stream0, stream_end;      // the streams this launch covers
    unsigned long long sample_begin, sample_end; // the slice of every stream this launch covers (multiples of the tile)
    int first_chunk;                   // start from reset_sdr_flow() state instead of the saved one
    struct StreamState *state;         // per-stream carried state between launches of one batch
    int use_mag, enable_fm, fpdm;
    int want_stages; // the FM stage array is wanted for every sample (fm_out)
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
    unsigned *counters; // [0] packages, [1] pool entries, [2] overflow flag, [4..] statistics
    int16_t *am;               // k_front's output (repaired in place where a tile did not fit its predecessor)
    ChunkInfo const *chunks;   // bounds of every 64-sample chunk of `am`
    int16_t *fm_out;           // optional stage dump, indexed by offsets[s]/SS + n
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
    int pri = 0, prq = 0; // IQ in front of the batch (zero in front of the stream: reset demod state)
    if (jb.fm_on && a > 0) {
        uint8_t const *g = jb.src + (a - 1) * SS;
        if (SS == 2) {
            pri = (int)(g[0] ^ (jb.flip & 0xff)) - 128;
            prq = (int)(g[1] ^ (jb.flip & 0xff)) - 128;
        } else {
            uint32_t w = *reinterpret_cast<uint32_t const *>(g) ^ jb.flip;
            pri = (int)(int16_t)(w & 0xffff);
            prq = (int)(int16_t)(w >> 16);
        }
    }
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
// (the stream start, or sm.fm_pos).  Monotone filters only.  Leaves the state in sm.fm_pos / fm_y / fm_xf.
template <int SS>
__device__ R4_NOINLINE void fm_cold(FmJob const &jb, WarpSmem &sm, unsigned long long pos)
{
    constexpr int SPL = 16 / SS;
    int const lane = threadIdx.x & 31;
    unsigned long long const known = sm.fm_pos; // state known here (always <= pos when used)
    for (unsigned long long K = 64;; K *= 4) {
        unsigned long long a = pos > K ? (pos - K) / SPL * SPL : 0;
        bool exact_start = a == 0;
        int lo, hi, fp;
        if (known <= pos && known >= a) { // reach back to the known state instead
            a = known;
            exact_start = true;
        }
        if (exact_start) {
            lo = hi = a == known ? sm.fm_y : 0;
            fp = a == known ? sm.fm_xf : 0;
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
                sm.fm_pos = pos;
                sm.fm_y = lo;
                sm.fm_xf = fp;
                sm.win_n = 0;
            }
            __syncwarp();
            return;
        }
        // not met: exactly constant input parks the two ends on different fixed points of the floor map
    }
}

// FM of the window [w0, w0 + n) (n <= kFmWin, w0 a multiple of SPL) from the exact state in sm.fm_* which
// must be the one in front of w0.  Advances sm.fm_pos to w0 + n.
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
            y = sm.fm_y;
            fp = sm.fm_xf;
        } else {
            fp = (int)sm.xf[fm_pidx(start - 1)];
            y = SS == 2 ? fp : fp; // the low-pass has unit gain: its state is near its input
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
            sm.fm_y = ye;
            sm.fm_xf = fe;
        }
    }
    if (lane == 0) {
        sm.fm_pos = w0 + n;
        sm.win0 = w0;
        sm.win_n = n;
    }
    __syncwarp();
    if (jb.fm_out) { // stage dump
        for (int i = lane; i < n; i += 32) jb.fm_out[w0 + i] = (int16_t)sm.fm[fm_pidx(i)];
    }
}

// Make the window that holds sample `pos` current (lazy mode): continue the previous window when it ends
// close in front, rebuild the state otherwise.
template <int SS>
__device__ R4_NOINLINE void fm_demand(FmJob const &jb, WarpSmem &sm, unsigned long long pos, unsigned long long limit)
{
    constexpr int SPL = 16 / SS;
    unsigned long long w0 = pos / SPL * SPL;
    if (jb.fm_on) {
        unsigned long long const have = sm.fm_pos;
        if (have > w0 || w0 - have > 2 * kFmWin) {
            fm_cold<SS>(jb, sm, w0);
        } else {
            while (sm.fm_pos + kFmWin <= w0) fm_window<SS>(jb, sm, sm.fm_pos, kFmWin); // walk up to it
            w0 = sm.fm_pos;
        }
    }
    unsigned long long end = w0 + kFmWin < limit ? w0 + kFmWin : limit;
    fm_window<SS>(jb, sm, w0, (int)(end - w0));
}

// The window for the detector walk at tile [t0, t0 + nv_tile): on demand (lazy), or re-made from the start
// states the tile pass kept (eager mode: windows are aligned, the end-of-tile state is put back afterwards).
template <int SS>
__device__ R4_NOINLINE void fm_for_walk(FmJob const &jb, WarpSmem &sm, unsigned long long pos, unsigned long long t0,
        int nv_tile, bool lazy)
{
    int const lane = threadIdx.x & 31;
    if (lazy) {
        fm_demand<SS>(jb, sm, pos, t0 + (unsigned long long)nv_tile);
        return;
    }
    int const w = (int)(pos - t0) / kFmWin;
    if (lane == 0) {
        sm.fm_y = sm.tile_state_y[w];
        sm.fm_xf = sm.tile_state_xf[w];
        sm.fm_pos = t0 + (unsigned long long)w * kFmWin;
    }
    __syncwarp();
    FmJob quiet = jb;
    quiet.fm_out = nullptr;
    int const cnt = nv_tile - w * kFmWin < kFmWin ? nv_tile - w * kFmWin : kFmWin;
    fm_window<SS>(quiet, sm, t0 + (unsigned long long)w * kFmWin, cnt);
    if (lane == 0) {
        sm.fm_pos = sm.tile_end_pos;
        sm.fm_y = sm.tile_end_y;
        sm.fm_xf = sm.tile_end_xf;
    }
    __syncwarp();
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
            while (cnt) {
                if (!(sm.win_n > 0 && pos >= sm.win0 && pos < sm.win0 + (unsigned long long)sm.win_n))
                    fm_demand<SS>(jb, sm, pos, jb.N);
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

// eager FM mode: put the contiguous end-of-tile filter state back after windows were (re-)made out of order
__device__ __forceinline__ void restore_tile_end(WarpSmem &sm)
{
    __syncwarp();
    if ((threadIdx.x & 31) == 0 && !sm.wc.lazy_fm) {
        sm.fm_pos = sm.tile_end_pos;
        sm.fm_y = sm.tile_end_y;
        sm.fm_xf = sm.tile_end_xf;
    }
    __syncwarp();
}

// everything logged so far into the exact value ws.d.ook_f1 (state in shared memory)
template <int SS>
__device__ R4_NOINLINE void walk_f1_fold(WarpSmem &sm)
{
    __syncwarp();
    int const g = f1_evaluate<SS>(sm.wc.jb, sm, sm.wc.log, sm.ws.d.start_abs, sm.ws.d.ook_f1, sm.ws.log_n, sm.ws.log_start,
            sm.ws.log_count);
    restore_tile_end(sm);
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
        idx = atomicAdd(&wc.counters[0], 1u);
        off = atomicAdd(&wc.counters[1], cnt);
    }
    idx = __shfl_sync(0xffffffffu, idx, 0);
    off = __shfl_sync(0xffffffffu, off, 0);
    bool fits = idx < wc.pkg_cap && (unsigned long long)off + cnt <= wc.pool_cap;
    if (!fits) {
        if (lane == 0) atomicOr(&wc.counters[2], 1u);
    } else {
        __syncwarp();
        int const *sp = type == 1 ? tr.ook_pulse : tr.fsk_pulse;
        int const *sg = type == 1 ? tr.ook_gap : tr.fsk_gap;
        for (unsigned i = lane; i < cnt; i += 32) {
            wc.pulse_pool[off + i] = sp[i];
            wc.gap_pool[off + i] = sg[i];
        }
        if (lane == 0) {
            unsigned long long blk = flush ? (N + wc.block_samples - 1) / wc.block_samples : pos / wc.block_samples;
            unsigned long long bstart = blk * wc.block_samples;
            unsigned long long blen = flush ? 0 : (N - bstart < wc.block_samples ? N - bstart : wc.block_samples);
            r433b_package k;
            k.stream = wc.stream;
            k.seq = seq;
            k.type = type;
            k.block = (int)blk;
            k.offset = h.offset;
            k.end_pos = pos;
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

__device__ __forceinline__ int am_tile_at(uint16_t const *am16, int n) { return (int)am16[(n >> 6) * (2 * kAmStride) + (n & 63)]; }

// IDLE from tile sample n on: only the noise-floor tracker moves.  Returns the first sample it could not take
// (a trigger is conceivable there, or the tracker leaves its +-1 regime): the generic step looks at that one.
__device__ R4_NOINLINE int idle_run(WarpSmem &sm, int n)
{
    constexpr int C = kChunk;
    int const lane = threadIdx.x & 31;
    uint16_t const *am16 = reinterpret_cast<uint16_t const *>(sm.am);
    __syncwarp();
    struct {
        int low, high, lead_in;
    } d = {sm.ws.d.low, sm.ws.d.high, sm.ws.d.lead_in};
    Levels const lv = sm.wc.lv;
    int const nv_tile = sm.ws.nv_tile;
    auto am_at = [&](int i) -> int { return am_tile_at(am16, i); };

    // IDLE over a long stretch, lane-parallel: see the comment in the file header and below.
    // While |am - low| < 1024 the tracker is low += (am > low) ? +1 : -1, so low keeps the parity of
    // (low0 + samples seen) and two trajectories of equal parity never cross and merge once the data
    // passes between them: lane l takes chunk l, starts from a bracket [lo, hi] of the right parity that
    // provably contains the true value, pushes both ends through its chunk and hands them to the next
    // lane until every bracket has collapsed.  Chunks in which a trigger is conceivable (or
    // |am - low| could reach 1024) end the stretch.
    auto idle_tile = [&](int n) -> int {
        if (nv_tile - n < 2 * C) return 0;
        {
            int hs = lv.ratio * d.low;
            if (hs < lv.min_high) hs = lv.min_high;
            if (d.high != hs) return 0;
        }
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
        int Lmin = d.low < pmin - 1 ? d.low : pmin - 1;
        int Lmax = d.low > pmax ? d.low : pmax;
        int hmin = lv.ratio * Lmin;
        if (hmin < lv.min_high) hmin = lv.min_high;
        Thresholds th = det_thresholds(Lmin, hmin, lv);
        bool const armed = d.lead_in + (nv_tile - n) > kLeadIn;
        bool ok = in_region && !(armed && cmax > th.up) && (pmax - Lmin < 1024) && (Lmax - pmin < 1024);
        unsigned bad = ~__ballot_sync(0xffffffffu, ok) & (0xffffffffu << c0);
        int const e = bad ? __ffs(bad) - 1 : 32; // chunks c0 .. e-1 form the stretch
        if (e - c0 < 2) return 0;
        int const RLmin = __shfl_sync(0xffffffffu, Lmin, e - 1);
        int const RLmax = __shfl_sync(0xffffffffu, Lmax, e - 1);
        bool const act = lane >= c0 && lane < e;
        int const par = (d.low + (lane * C + k0 - n)) & 1; // parity of the true value at this lane's start
        // Start bracket.  Over K samples whose values lie in [m, M] the tracker climbs one per sample
        // until it is >= m - 1 and falls one per sample until it is <= M, so from any start in [A, B] it
        // ends in [min(A + K, m - 1), max(B - K, M)].  The chunk to the left has K = 64 samples (the first
        // chunk of the stretch may be partial: then the exact start value and its real length are used).
        int m1 = __shfl_up_sync(0xffffffffu, cmin, 1), M1 = __shfl_up_sync(0xffffffffu, cmax, 1);
        int K1 = __shfl_up_sync(0xffffffffu, k1 - k0, 1);
        int lo, hi;
        if (lane == c0 + 1) {
            lo = d.low + K1 < m1 - 1 ? d.low + K1 : m1 - 1;
            hi = d.low - K1 > M1 ? d.low - K1 : M1;
        } else {
            lo = RLmin + K1 < m1 - 1 ? RLmin + K1 : m1 - 1;
            hi = RLmax - K1 > M1 ? RLmax - K1 : M1;
        }
        lo = lo < RLmin ? RLmin : lo;
        hi = hi > RLmax ? RLmax : hi;
        lo -= (lo - par) & 1;
        hi += (hi - par) & 1;
        if (lane == c0) lo = hi = d.low;
        uint16_t const *chunk = am16 + lane * (2 * kAmStride);
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
            // the true value lies inside every bracket: collapsed end brackets are the true values
            if (__all_sync(0xffffffffu, !act || elo == ehi)) {
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
        int hh = lv.ratio * d.low;
        d.high = hh < lv.min_high ? lv.min_high : hh;
        int li = d.lead_in + len;
        d.lead_in = li > kLeadIn + 1 ? kLeadIn + 1 : li;
        return len;
    };

    // IDLE: only the noise-floor tracker moves (src/pulse_detect.c:325-334).  While
    // |am - low| < 1024 it is low += (am > low) ? +1 : -1; with q = low + j that is
    // q += 2 * (am_j + j > q): two dependent instructions per sample.
    auto idle_fast = [&](int n) -> int {
        int cnt = nv_tile - n < 32 ? nv_tile - n : 32;
        int hs = lv.ratio * d.low;
        if (hs < lv.min_high) hs = lv.min_high;
        if (d.high != hs) return 0; // first IDLE sample after a package: not yet re-derived
        int a = lane < cnt ? am_at(n + lane) : -32768;
        int lmin = d.low - cnt;
        int hmin = lv.ratio * lmin;
        if (hmin < lv.min_high) hmin = lv.min_high;
        Thresholds th = det_thresholds(lmin, hmin, lv); // lowest trigger level reachable in this chunk
        bool armed = d.lead_in + cnt - 1 > kLeadIn;
        bool stop = lane < cnt && ((armed && a > th.up) || (a - lmin >= 1024) || (d.low + cnt - a >= 1024));
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
        int hh = lv.ratio * d.low;
        d.high = hh < lv.min_high ? lv.min_high : hh;
        int li = d.lead_in + cnt;
        d.lead_in = li > kLeadIn + 1 ? kLeadIn + 1 : li;
        return cnt;
    };


    while (n < nv_tile) {
        int adv = idle_tile(n);
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
                int const aq = a >> 6; // am >= 0
                int const top = __reduce_max_sync(0xffffffffu, lane < cnt ? aq : 0); // one REDUX each
                    int hmax = 64 * top + 63;
                hmax = h > hmax ? h : hmax;
                unsigned const m = __ballot_sync(0xffffffffu, lane < cnt && a < det_thresholds(low, hmax, lv).down);
                if (m) cnt = __ffs(m) - 1;
                if (cnt) {
                    __syncwarp();
                    sm.q[lane] = aq;
                    __syncwarp();
                    // h >= min_high >= 0 here, so h / 64 == h >> 6.  Eight steps per trip, the loops kept rolled: seven
                // warps per scheduler share an instruction cache of a few hundred instructions.
                // q >= 0, so one step takes at most h >> 6 off, and less from a lower h: after k steps h is still
                // >= h0 - k (h0 >> 6).  If that stays >= min_high over the whole stretch the clamp of :363 cannot act
                // and is left out of the dependency chain.
                int4 const *qp = reinterpret_cast<int4 const *>(sm.q);
                int trips = cnt >> 3;
#define R4_STEP(q) h += (q) - (int)((unsigned)h >> 6)
#define R4_STEP_CLAMPED(q) h = max(h + (q) - (int)((unsigned)h >> 6), minh)
#if R4_REC == 2
                if (h - cnt * (int)((unsigned)h >> 6) >= minh) {
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
#elif R4_REC == 1
#pragma unroll 1
                for (; trips > 0; --trips, qp += 2) {
                    int4 const b = qp[0], c = qp[1];
                    if (h - 8 * (int)((unsigned)h >> 6) >= minh) {
                        R4_STEP(b.x); R4_STEP(b.y); R4_STEP(b.z); R4_STEP(b.w);
                        R4_STEP(c.x); R4_STEP(c.y); R4_STEP(c.z); R4_STEP(c.w);
                    } else {
                        R4_STEP_CLAMPED(b.x); R4_STEP_CLAMPED(b.y); R4_STEP_CLAMPED(b.z); R4_STEP_CLAMPED(b.w);
                        R4_STEP_CLAMPED(c.x); R4_STEP_CLAMPED(c.y); R4_STEP_CLAMPED(c.z); R4_STEP_CLAMPED(c.w);
                    }
                }
#else
#pragma unroll 1
                for (; trips > 0; --trips, qp += 2) {
                    int4 const b = qp[0], c = qp[1];
                    R4_STEP_CLAMPED(b.x); R4_STEP_CLAMPED(b.y); R4_STEP_CLAMPED(b.z); R4_STEP_CLAMPED(b.w);
                    R4_STEP_CLAMPED(c.x); R4_STEP_CLAMPED(c.y); R4_STEP_CLAMPED(c.z); R4_STEP_CLAMPED(c.w);
                }
#endif
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
                        h += (aj >> 6) - (int)((unsigned)h >> 6);
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
    bool const lazy_fm = sm.wc.lazy_fm != 0;
    int const nv_tile = sm.ws.nv_tile;
    unsigned long long const t0 = sm.ws.t0;
    WarpCtx cx;
    cx.lane = lane;
    cx.nlanes = 32;
#pragma unroll 1
    while (n < nv_tile) {
        unsigned long long const pos = t0 + (unsigned long long)n;
        if (!(sm.win_n > 0 && pos >= sm.win0 && pos < sm.win0 + (unsigned long long)sm.win_n))
            fm_for_walk<SS>(sm.wc.jb, sm, pos, t0, nv_tile, lazy_fm);
        int cnt = nv_tile - n < 32 ? nv_tile - n : 32;
        int const in_win = (int)(sm.win0 + (unsigned long long)sm.win_n - pos);
        cnt = cnt < in_win ? cnt : in_win;
        int const a = lane < cnt ? am_tile_at(am16, n + lane) : 32767;
        int const f = lane < cnt ? (int)(int16_t)sm.fm[fm_pidx((int)(pos - sm.win0) + lane)] : 0;
        int const aq = a >> 6;
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
    bool const defer_f1 = sm.wc.defer_f1 != 0, lazy_fm = sm.wc.lazy_fm != 0;
    int const nv_tile = sm.ws.nv_tile;
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
    // FM of tile sample i: make the window that holds it current first
    auto fm_need = [&](int i) {
        unsigned long long pos = t0 + (unsigned long long)i;
        if (sm.win_n > 0 && pos >= sm.win0 && pos < sm.win0 + (unsigned long long)sm.win_n) return;
        fm_for_walk<SS>(sm.wc.jb, sm, pos, t0, nv_tile, lazy_fm);
    };
    auto fm_at = [&](int i) -> int { return (int)(int16_t)sm.fm[fm_pidx((int)(t0 + (unsigned long long)i - sm.win0))]; };

    // inside a first pulse (and its GAP_START) the FSK sub-detector and the undeferred estimate read FM
    bool const first = d.ook_n == 0 && (d.st == kPulse || d.st == kGapStart);
    bool const wants_fm = first || (d.st == kPulse && !defer_f1);
    if (wants_fm) fm_need(n);
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
    bool const fm_on = p.enable_fm != 0;

    unsigned long long const byte0 = p.offsets[s];
    unsigned long long const N = (p.lengths ? p.lengths[s] : p.offsets[s + 1] - byte0) / SS;
    uint8_t const *const src = p.data + byte0;
    int16_t *const am_stream = p.am + p.am_offsets[s];
    ChunkInfo const *const chunk_stream = p.chunks + p.am_offsets[s] / kChunk;
    // FM windows on demand need the rigorous state rebuild (monotone filter); the stage dump wants every sample
    bool const lazy_fm = !fm_on || (p.wrap_free && !p.want_stages);
    // the deferred carrier estimate re-makes FM for logged samples later: needs the state rebuild as well
    bool const defer_f1 = !fm_on || p.wrap_free != 0;

    int y_am = 0; // the last AM value of the previous tile: the AM filter state (reset_sdr_flow(): zero)
    int flushed = 0;
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
        wc.jb.fm_out = p.fm_out ? p.fm_out + byte0 / SS : nullptr;
        wc.tr.ook_pulse = p.train_scratch + (size_t)s * kTrainInts;
        wc.tr.ook_gap = wc.tr.ook_pulse + kMaxPulses;
        wc.tr.fsk_pulse = wc.tr.ook_gap + kMaxPulses;
        wc.tr.fsk_gap = wc.tr.fsk_pulse + kMaxPulses;
        wc.log = p.log_scratch + (size_t)s * kLogCap * 2;
        wc.lv = p.lv;
        wc.per_ms = (int)(p.rate / 1000);
        wc.fpdm = p.fpdm;
        wc.lazy_fm = lazy_fm;
        wc.defer_f1 = defer_f1;
        wc.stream = s;
        wc.block_samples = p.block_samples;
        wc.pkgs = p.pkgs;
        wc.pulse_pool = p.pulse_pool;
        wc.gap_pool = p.gap_pool;
        wc.pkg_cap = p.pkg_cap;
        wc.pool_cap = p.pool_cap;
        wc.counters = p.counters;
        WalkState &ws = sm.ws;
        ws.pend_type = 0;
        ws.pend_pos = 0;
        ws.t0 = 0;
        ws.nv_tile = 0;
        if (p.first_chunk) {
            det_reset(ws.d);
            ws.d.ook_hw = ws.d.fsk_hw = kMaxPulses; // scratch is not assumed to be zero: first package clears it
            ws.log_n = ws.log_start = ws.log_count = 0;
            ws.seq = 0;
            sm.fm_pos = 0;
            sm.fm_y = sm.fm_xf = 0;
        } else {
            StreamState const &ss = p.state[s];
            ws.d = ss.d;
            ws.seq = ss.seq;
            ws.log_n = ss.log_n;
            ws.log_start = ss.last_start;
            ws.log_count = ss.last_count;
            sm.fm_pos = ss.fm_pos;
            sm.fm_y = ss.fm_y;
            sm.fm_xf = ss.fm_xf;
        }
        sm.win0 = 0;
        sm.win_n = 0;
    }
    if (!p.first_chunk) {
        y_am = p.state[s].y_am;
        flushed = p.state[s].flushed;
    }
    __syncwarp();

    int const a1 = p.lpf_a1, b0 = p.lpf_b0;

    for (unsigned long long t0 = p.sample_begin; t0 < p.sample_end && t0 < N; t0 += T) {
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
            int x0 = 0, xm = 0;
            if (t0 != 0) {
                x0 = env_at<SS>(src, t0, p.flip, p.use_mag);
                xm = env_at<SS>(src, t0 - 1, p.flip, p.use_mag);
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
            // hand-over check (see the file header): the first tile of a stream starts from the reset state in k_front
            if (t0 != 0) {
                // the reference keeps x[-1] as int16 across block calls (src/baseband.c:167)
                if (t0 % p.block_samples == 0) xm = (int)(int16_t)xm;
                int const expect = iir16_nowrap(y_am, a1, b0, x0 + xm);
                if (expect != (int)(int16_t)am16[0]) {
                    am_repair<SS>(sm, src, t0, nv_tile, y_am, xm, a1, b0, p.flip, p.use_mag, am_stream + t0);
                    if (lane == 0) atomicAdd(&p.counters[5], 1u);
                }
            }
        }
        y_am = am_tile_at(am16, nv_tile - 1);
        // ---- FM for the whole tile when it cannot be made on demand -----------------------------
        if (!lazy_fm || (!fm_on && p.fm_out)) {
            for (int w = 0; w * kFmWin < nv_tile; ++w) {
                if (lane == 0) {
                    sm.tile_state_y[w] = sm.fm_y;
                    sm.tile_state_xf[w] = sm.fm_xf;
                }
                __syncwarp();
                int n = nv_tile - w * kFmWin < kFmWin ? nv_tile - w * kFmWin : kFmWin;
                fm_window<SS>(sm.wc.jb, sm, t0 + (unsigned long long)w * kFmWin, n);
            }
            if (lane == 0) {
                sm.tile_end_pos = sm.fm_pos;
                sm.tile_end_y = sm.fm_y;
                sm.tile_end_xf = sm.fm_xf;
            }
            __syncwarp();
        }

        // ---- package detector over the tile (warp-uniform), phase by phase ------------------------
        if (t0 % p.block_samples == 0) walk_call_boundary(sm);
        for (int n = 0; n < nv_tile;) {
            int const st = sm.ws.d.st;
            int m = n;
            if (st == kIdle)
                m = idle_run(sm, n);
            else if (defer_f1 && !sm.ws.d.eop_flag && (sm.ws.d.ook_n != 0 || st == kGap))
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

    // flush_sdr_flow(): len == 0 call(s) at the end of the file, in the launch that reaches it
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
        ss.fm_pos = sm.fm_pos;
        ss.fm_y = sm.fm_y;
        ss.fm_xf = sm.fm_xf;
        ss.log_n = sm.ws.log_n;
        ss.last_start = sm.ws.log_start;
        ss.last_count = sm.ws.log_count;
        ss.seq = sm.ws.seq;
        ss.flushed = flushed;
    }
}

} // namespace r433b
