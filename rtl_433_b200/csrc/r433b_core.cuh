// r433b_core.cuh -- per-sample arithmetic and state machines of the IQ -> pulse-train path.
//
// Everything here is a __host__ __device__ inline so the same code that runs inside the
// sm_90a kernels (r433b_kernels.cu) can be exercised on the CPU by tests/ (host_core.cpp);
// the product path itself only ever calls these from device code.
//
// The detector is written in STREAMING form: one call per sample with an absolute sample
// index, no notion of "blocks".  The reference processes fixed blocks and re-enters its
// detector after every package (src/pulse_detect.c:199-483); the observable consequences of
// that call structure are applied by the caller through det_call_boundary().
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define R4_HD __host__ __device__ __forceinline__
#define R4_HD_COLD __host__ __device__ __noinline__
#else
#define R4_HD inline
#define R4_HD_COLD inline
#endif

namespace r433b {

constexpr int kMaxPulses = 1200;     // include/pulse_data.h:21 PD_MAX_PULSES
constexpr int kMinPulses = 16;       // :22 PD_MIN_PULSES
constexpr int kMinPulseSamples = 10; // :23 PD_MIN_PULSE_SAMPLES
constexpr int kLeadIn = 1024;        // src/pulse_detect.c:27 OOK_EST_LOW_RATIO

// ------------------------------------------------------------------ sample maps --------

// src/baseband.c:22-45: squared distance from 127 (not 128)
R4_HD int env_cu8(int i, int q)
{
    int di = 127 - i, dq = 127 - q;
    return di * di + dq * dq;
}

// src/baseband.c:65-79
R4_HD int mag_cu8(int i, int q)
{
    int a = i - 128, b = q - 128;
    a = a < 0 ? -a : a;
    b = b < 0 ? -b : b;
    int hi = a > b ? a : b, lo = a > b ? b : a;
    return (122 * hi + 51 * lo) & 0xffff;
}

// src/baseband.c:96-110
R4_HD int mag_cs16(int i, int q)
{
    unsigned a = (unsigned)(i < 0 ? -i : i), b = (unsigned)(q < 0 ? -q : q);
    unsigned hi = a > b ? a : b, lo = a > b ? b : a;
    return (int)(((122u * hi + 51u * lo) >> 8) & 0xffffu);
}

// t / den with C semantics (truncation toward zero) for |t| < 2^30, 1 <= den <= 2^17 and
// |t / den| < 2^14.  On the device: float reciprocal estimate (error < 0.01 in the quotient)
// plus one exact integer correction step, instead of the generic 32-bit division sequence.
R4_HD int div_trunc_small(int t, int den)
{
#ifdef __CUDA_ARCH__
    unsigned u = (unsigned)(t < 0 ? -t : t);
    int q = (int)(__fmul_rn((float)u, __frcp_rn((float)den)));
    int r = (int)u - q * den;
    if (r < 0)
        q -= 1;
    else if (r >= den)
        q += 1;
    return t < 0 ? -q : q;
#else
    return t / den;
#endif
}

// src/baseband.c:181-202: pi == 32767, truncating division, (0,0) -> 0
R4_HD int atan16(int y, int x)
{
    int ay = y < 0 ? -y : y;
    if ((x | y) == 0) return 0;
    int num, den, base;
    if (x >= 0) {
        den = ay + x;
        num = x - ay;
        base = 8191;
    } else {
        den = ay - x;
        num = x + ay;
        base = 24575;
    }
    // den >= 1 here: it is 0 only for x == y == 0; |num| <= den <= 65536
    int ang = base - div_trunc_small(8191 * num, den);
    return (int)(int16_t)(y < 0 ? -ang : ang);
}

// t / den with C semantics for |t| < 2^62, 1 <= den < 2^33 and |t / den| < 2^30.  On the
// device: double-precision reciprocal estimate (quotient error < 2^-20) plus one exact 64-bit
// correction step, instead of the ~100-instruction generic 64-bit division.
R4_HD long long div_trunc_big(long long t, long long den)
{
#ifdef __CUDA_ARCH__
    unsigned long long u = (unsigned long long)(t < 0 ? -t : t);
    long long q = (long long)__dmul_rn((double)u, __drcp_rn((double)den));
    long long r = (long long)u - q * den;
    if (r < 0)
        q -= 1;
    else if (r >= den)
        q += 1;
    return t < 0 ? -q : q;
#else
    return t / den;
#endif
}

// src/baseband.c:281-300: pi == INT32_MAX, no (0,0) case, arguments already narrowed to int32
R4_HD int atan32(int y, int x)
{
    long long const q = 536870911ll, q3 = 1610612735ll;
    long long ay = (long long)(int)(y < 0 ? (int)(0u - (unsigned)y) : y);
    long long ang;
    if (x >= 0) {
        long long d = ay + x;
        if (d == 0) d = 1;
        ang = q - div_trunc_big(q * (x - ay), d);
    } else {
        long long d = ay - x;
        if (d == 0) d = 1;
        ang = q3 - div_trunc_big(q * (x + ay), d);
    }
    return (int)(y < 0 ? -ang : ang);
}

// one step of the Q0.15 first-order low-pass shared by the AM filter (src/baseband.c:161-163)
// and the cu8 FM filter (:263): y' = int16((a1*y + b0*(x0 + x1)) >> 14)
R4_HD int iir16(int y, int a1, int b0, int xsum)
{
    return (int)(int16_t)((a1 * y + b0 * xsum) >> 14);
}

// the same step when the host has proved the state can never leave the int16 range
// (coefficients non-negative with a1 + 2*b0 <= 16384): the int16 store is then the identity
R4_HD int iir16_nowrap(int y, int a1, int b0, int xsum)
{
    return (a1 * y + b0 * xsum) >> 14;
}

// the Q0.30 variant of the cs16 FM filter, int64 accumulate (src/baseband.c:357)
R4_HD int iir32(int y, long long a1, long long b0, long long xsum)
{
    return (int)((a1 * (long long)y + b0 * xsum) >> 30);
}

// --------------------------------------------------------------------- detector ---------

struct Levels {
    int fixed_high; // src/pulse_detect.c:32, 0 = adaptive
    int min_high;   // :33
    int ratio;      // :34
    int max_high;   // :24 OOK_MAX_HIGH_LEVEL
    int monotone;   // derived_high() is non-decreasing in `low` over its whole range (compute_levels proves it)
};

// `high` as IDLE derives it from `low` (src/pulse_detect.c:331-332).  ratio * low is int multiplication in the
// reference: above min_snr ~48 dB (envelope) it wraps in 32 bits, as it does on the hardware the reference runs on.
R4_HD int derived_high(int low, Levels const &lv)
{
    int const h = (int)((unsigned)lv.ratio * (unsigned)low);
    return h < lv.min_high ? lv.min_high : h;
}

enum { kIdle = 0, kPulse = 1, kGapStart = 2, kGap = 3 };
enum { kFskInit = 0, kFskHigh = 1, kFskLow = 2, kFskErr = 3 };

// storage of the two pulse trains of one stream (global memory on the device)
struct Trains {
    int *ook_pulse, *ook_gap, *fsk_pulse, *fsk_gap; // kMaxPulses each
};

struct DetState {
    int st, run, longest, lead_in, low, high;
    int eop_flag; // eop_on_spurious, a local of the reference call: cleared at call boundaries
    // OOK train header
    unsigned ook_n;
    int ook_f1;
    int last_pulse;
    unsigned ook_hw; // entries [0, hw) may be non-zero
    // FSK train header
    unsigned fsk_n;
    unsigned long long fsk_offset;
    unsigned fsk_hw;
    // where the current package started (absolute sample index)
    unsigned long long start_abs;
    // FSK sub-detector, include/pulse_detect_fsk.h:23-41
    unsigned fk_len;
    int fk_st, fk_f1, fk_f2, fk_vmax, fk_vmin, fk_skip;
};

R4_HD void fsk_reset(DetState &d)
{
    d.fk_len = 0;
    d.fk_st = kFskInit;
    d.fk_f1 = d.fk_f2 = 0;
    d.fk_vmax = -32768;
    d.fk_vmin = 32767;
    d.fk_skip = 40;
}

R4_HD void det_reset(DetState &d) // src/pulse_detect.c:74-84 (+ freshly zeroed pulse_data)
{
    d.st = kIdle;
    d.run = d.longest = d.lead_in = d.low = d.high = 0;
    d.eop_flag = 0;
    d.ook_n = 0;
    d.ook_f1 = 0;
    d.last_pulse = 0;
    d.fsk_n = 0;
    d.fsk_offset = 0;
    d.start_abs = 0;
    fsk_reset(d);
}

// What every entry into pulse_detect_package() does before looking at samples
// (src/pulse_detect.c:283, :291): applies at block starts and after each returned package.
R4_HD void det_call_boundary(DetState &d, Levels const &lv)
{
    if (d.high < lv.min_high) d.high = lv.min_high;
    d.eop_flag = 0;
}

R4_HD void put(int *arr, unsigned &hw, unsigned i, int v)
{
    arr[i] = v;
    if (i + 1 > hw) hw = i + 1;
}

// src/pulse_data.c:27-34 on the FSK train (offset grows by the COUNT: kept quirk).  The memory move is out
// of line (cold, and the sub-detectors that call it are inlined several times); no state escapes into it.
template <class Ctx>
R4_HD_COLD void fsk_shift_move(int *pulse, int *gap, Ctx cx)
{
    int const half = kMaxPulses / 2;
    cx.sync();
    for (int i = cx.lane; i < half; i += cx.nlanes) {
        pulse[i] = pulse[i + half];
        gap[i] = gap[i + half];
    }
    cx.sync();
}
template <class D, class Ctx>
R4_HD void fsk_shift(D &d, Trains const &t, Ctx &cx)
{
    fsk_shift_move(t.fsk_pulse, t.fsk_gap, cx);
    d.fsk_n -= kMaxPulses / 2;
    d.fsk_offset += kMaxPulses / 2;
    d.fsk_hw = kMaxPulses;
}

// A train entry read back by a warp-uniform step.  Every lane writes the same entries, and nothing but a collective
// keeps the lanes of a warp at the same sample: without the first sync a lane could read an entry before a slower lane
// has written it for this sample, without the second a faster lane could overwrite it for a later sample before a
// slower one has read it (first_run feeds the FSK sub-detector up to 32 samples per trip with no collective between).
template <class Ctx>
R4_HD int train_read(int const *arr, unsigned i, Ctx &cx)
{
    cx.sync();
    int const v = arr[i];
    cx.sync();
    return v;
}

// src/pulse_detect_fsk.c:34-141
template <class D, class Ctx>
R4_HD void fsk_classic(D &d, Trains const &t, int v, Ctx &cx)
{
    int d1 = v - d.fk_f1, d2 = v - d.fk_f2;
    d1 = d1 < 0 ? -d1 : d1;
    d2 = d2 < 0 ? -d2 : d2;
    d.fk_len += 1;
    if (d.fk_st == kFskInit) {
        if (d.fk_len < (unsigned)kMinPulseSamples) {
            d.fk_f1 = d.fk_f1 / 2 + v / 2;
        } else if (d1 > 3000) {
            if (v > d.fk_f1) {
                d.fk_st = kFskHigh;
                d.fk_f2 = d.fk_f1;
                d.fk_f1 = v;
                put(t.fsk_pulse, d.fsk_hw, 0, 0);
                put(t.fsk_gap, d.fsk_hw, 0, (int)d.fk_len);
                d.fsk_n += 1;
                d.fk_len = 0;
            } else {
                d.fk_st = kFskLow;
                d.fk_f2 = v;
                put(t.fsk_pulse, d.fsk_hw, 0, (int)d.fk_len);
                d.fk_len = 0;
            }
        } else {
            d.fk_f1 += v / 16 - d.fk_f1 / 16;
        }
    } else if (d.fk_st == kFskHigh) {
        if (d1 > d2) {
            d.fk_st = kFskLow;
            if (d.fk_len >= (unsigned)kMinPulseSamples) {
                put(t.fsk_pulse, d.fsk_hw, d.fsk_n, (int)d.fk_len);
                d.fk_len = 0;
            } else {
                d.fk_len += (unsigned)train_read(t.fsk_gap, d.fsk_n - 1, cx);
                d.fsk_n -= 1;
                if (d.fsk_n == 0 && train_read(t.fsk_pulse, 0, cx) == 0) {
                    d.fk_f1 = d.fk_f2;
                    d.fk_st = kFskInit;
                }
            }
        } else {
            int div = v > d.fk_f1 ? 16 : 64;
            d.fk_f1 += v / div - d.fk_f1 / div;
        }
    } else if (d.fk_st == kFskLow) {
        if (d2 > d1) {
            d.fk_st = kFskHigh;
            if (d.fk_len >= (unsigned)kMinPulseSamples) {
                put(t.fsk_gap, d.fsk_hw, d.fsk_n, (int)d.fk_len);
                d.fsk_n += 1;
                d.fk_len = 0;
                if (d.fsk_n >= (unsigned)kMaxPulses) fsk_shift(d, t, cx);
            } else {
                d.fk_len += (unsigned)train_read(t.fsk_pulse, d.fsk_n, cx);
                if (d.fsk_n == 0) d.fk_st = kFskInit;
            }
        } else {
            int div = v < d.fk_f2 ? 16 : 64;
            d.fk_f2 += v / div - d.fk_f2 / div;
        }
    }
}

// src/pulse_detect_fsk.c:143-156
R4_HD void fsk_wrap_up(DetState &d, Trains const &t)
{
    if (d.fsk_n >= (unsigned)kMaxPulses) return;
    d.fk_len += 1;
    if (d.fk_st == kFskHigh) {
        put(t.fsk_pulse, d.fsk_hw, d.fsk_n, (int)d.fk_len);
        put(t.fsk_gap, d.fsk_hw, d.fsk_n, 0);
    } else {
        put(t.fsk_gap, d.fsk_hw, d.fsk_n, (int)d.fk_len);
    }
    d.fsk_n += 1;
}

// src/pulse_detect_fsk.c:158-221 (int16 trackers; f1/f2 deliberately crossed, :192/:208)
template <class D, class Ctx>
R4_HD void fsk_minmax(D &d, Trains const &t, int v, Ctx &cx)
{
    if (d.fk_skip == 0) {
        if (v > d.fk_vmax) d.fk_vmax = v;
        if (v < d.fk_vmin) d.fk_vmin = v;
        int mid = (int)(int16_t)((d.fk_vmax + d.fk_vmin) / 2);
        if (v > mid) d.fk_vmax = (int)(int16_t)(d.fk_vmax - 10);
        if (v < mid) d.fk_vmin = (int)(int16_t)(d.fk_vmin + 10);
        d.fk_len += 1;
        if (d.fk_st == kFskInit) {
            d.fk_st = v > mid ? kFskHigh : kFskLow;
        } else if (d.fk_st == kFskHigh) {
            if (v < mid) {
                d.fk_st = kFskLow;
                put(t.fsk_pulse, d.fsk_hw, d.fsk_n, (int)d.fk_len);
                d.fk_len = 0;
            }
            d.fk_f2 += v / 64 - d.fk_f2 / 64;
        } else if (d.fk_st == kFskLow) {
            if (v > mid) {
                d.fk_st = kFskHigh;
                put(t.fsk_gap, d.fsk_hw, d.fsk_n, (int)d.fk_len);
                d.fsk_n += 1;
                d.fk_len = 0;
                if (d.fsk_n >= (unsigned)kMaxPulses) fsk_shift(d, t, cx);
            }
            d.fk_f1 += v / 64 - d.fk_f1 / 64;
        }
    }
    if (d.fk_skip > 0) d.fk_skip -= 1;
}

// the two levels the four states compare against (src/pulse_detect.c:300-304)
struct Thresholds {
    int up, down; // a > up: "above"; a < down: "below"
};

R4_HD Thresholds det_thresholds(int low, int high, Levels const &lv)
{
    int top = high < lv.max_high ? high : lv.max_high;
    int thr = (int)(int16_t)((low + top) / 2);
    if (lv.fixed_high != 0) thr = (int)(int16_t)lv.fixed_high;
    int hys = (int)(int16_t)(thr / 8);
    Thresholds r;
    r.up = thr + hys;
    r.down = thr - hys;
    return r;
}

// The lowest trigger level IDLE can reach while `low` stays >= lmin and `high` is derived from it (k_detect's IDLE
// shortcuts): `up` grows with `low` and with `high`, so it is the one at lmin where derived_high() is monotone
// (Levels::monotone), otherwise the one with `high` at its floor min_high
R4_HD int lowest_up(int lmin, Levels const &lv)
{
    return det_thresholds(lmin, lv.monotone ? derived_high(lmin, lv) : lv.min_high, lv).up;
}

// one IDLE sample that does not start a package (src/pulse_detect.c:325-334)
R4_HD void idle_track(DetState &d, Levels const &lv, int a)
{
    int delta = a - d.low;
    d.low += delta / 1024;
    d.low += delta > 0 ? 1 : -1;
    d.high = derived_high(d.low, lv);
    if (d.lead_in <= kLeadIn) d.lead_in += 1;
}

// package start (src/pulse_detect.c:311-323): both trains are cleared
template <class Ctx>
R4_HD void begin_package(DetState &d, Trains const &t, unsigned long long pos, Ctx &cx)
{
    cx.sync();
    for (unsigned i = cx.lane; i < d.ook_hw; i += cx.nlanes) {
        t.ook_pulse[i] = 0;
        t.ook_gap[i] = 0;
    }
    for (unsigned i = cx.lane; i < d.fsk_hw; i += cx.nlanes) {
        t.fsk_pulse[i] = 0;
        t.fsk_gap[i] = 0;
    }
    cx.sync();
    d.ook_hw = d.fsk_hw = 0;
    d.ook_n = d.fsk_n = 0;
    d.ook_f1 = 0;
    d.last_pulse = 0;
    d.start_abs = pos;
    d.fsk_offset = pos;
    d.run = 0;
    d.longest = 0;
    fsk_reset(d);
    d.st = kPulse;
}

// FSK hand-over (src/pulse_detect.c:387-410 / :239-253); estimates are read by the caller
R4_HD void close_fsk(DetState &d, Trains const &t, int fpdm)
{
    if (fpdm == 0) fsk_wrap_up(d, t);
    d.st = kIdle;
}

// One sample through the four-state machine (src/pulse_detect.c:293-476).
// Returns 0: sample consumed; 1: OOK package complete; 2: FSK package complete.
// On 1/2 the sample has NOT been consumed: the caller emits, applies det_call_boundary()
// and presents the same sample again (the reference returns before `data_counter += 1`).
//
// `defer_f1`: the carrier estimate of an OOK package (pulses->fsk_f1_est, :365) is only READ when the
// package is returned.  With defer_f1 the update is not applied after the first pulse; the return value
// carries kStepF1Deferred instead and the caller logs the sample (k_detect evaluates the estimate when the
// package ends, from the logged samples: r433b_detect.cuh).  `f` is then only looked at while
// ook_n == 0 (the FSK sub-detector and the estimate of the first pulse).
//
// Mode kStepLean compiles the FSK sub-detector out: valid whenever fsk_n <= 16 and ook_n != 0 or the state is IDLE / GAP.
// Mode kStepFirst only has the PULSE / GAP_START branches: valid inside a first pulse (ook_n == 0).  k_detect
// keeps the lean instance on its hot path and enters the other only inside first pulses; kStepAll is everything.
enum { kStepF1Deferred = 4 };
enum { kStepAll = 0, kStepLean = 1, kStepFirst = 2 };
template <int Mode = kStepAll, class Ctx>
R4_HD int det_step(DetState &d, Levels const &lv, Trains const &t, int a, int f, unsigned long long pos,
        int per_ms, int fpdm, Ctx &cx, bool defer_f1 = false)
{
    constexpr bool WithFsk = Mode != kStepLean;
    Thresholds th = det_thresholds(d.low, d.high, lv);
    bool const above = a > th.up;
    bool const below = a < th.down;
    if (Mode != kStepFirst && d.st == kIdle) {
        if (above && d.lead_in > kLeadIn)
            begin_package(d, t, pos, cx);
        else
            idle_track(d, lv, a);
        return 0;
    }
    d.run += 1;
    int deferred = 0;
    if (d.st == kPulse || d.st == kGapStart) {
        // the FSK sub-detector sees every sample of a first pulse and of the gap start behind it (:368-374, :414-420)
        bool const feed = WithFsk && d.ook_n == 0;
        if (d.st == kPulse) {
            if (below) {
                if (d.run < kMinPulseSamples) {
                    if (d.ook_n <= 1) {
                        d.st = kIdle;
                    } else {
                        d.eop_flag = 1;
                        d.st = kGap;
                    }
                } else {
                    put(t.ook_pulse, d.ook_hw, d.ook_n, d.run);
                    d.last_pulse = d.run;
                    if (d.run > d.longest) d.longest = d.run;
                    d.run = 0;
                    d.st = kGapStart;
                }
            } else {
                d.high += a / 64 - d.high / 64;
                if (d.high < lv.min_high) d.high = lv.min_high;
                if (defer_f1 && d.ook_n != 0)
                    deferred = kStepF1Deferred;
                else
                    d.ook_f1 += f / 64 - d.ook_f1 / 64;
            }
        } else {
            if (above) {
                d.run += d.last_pulse;
                d.st = kPulse;
            } else if (d.run >= kMinPulseSamples) {
                d.st = kGap;
                // only the first pulse and its GAP_START feed the FSK train, but that GAP_START feeds it once more on the
                // sample it moves to GAP: a later GAP_START can find fsk_n > 16 too (k_detect then keeps out of burst_run)
                if (WithFsk && d.fsk_n > (unsigned)kMinPulses) {
                    close_fsk(d, t, fpdm);
                    return 2;
                }
            }
        }
        if (feed) {
            if (fpdm == 0)
                fsk_classic(d, t, f, cx);
            else
                fsk_minmax(d, t, f, cx);
        }
        return deferred;
    }
    // kGap
    if (Mode == kStepFirst) return 0; // not reached: a first-pulse step is PULSE or GAP_START
    if (above) {
        put(t.ook_gap, d.ook_hw, d.ook_n, d.run);
        d.ook_n += 1;
        if (d.ook_n >= (unsigned)kMaxPulses) {
            d.st = kIdle;
            return 1;
        }
        d.run = 0;
        d.st = kPulse;
    }
    if (d.eop_flag || (d.run > 10 * d.longest && d.run > 10 * per_ms) || d.run > 100 * per_ms) {
        put(t.ook_gap, d.ook_hw, d.ook_n, d.run);
        d.ook_n += 1;
        d.st = kIdle;
        return 1;
    }
    return 0;
}

// End-of-input flush (src/pulse_detect.c:204-278).  Returns 0, 1 or 2 like det_step().
R4_HD int det_flush(DetState &d, Trains const &t, int fpdm)
{
    int st = d.st;
    if (st == kIdle) return 0;
    if (st == kPulse) {
        if (d.run < kMinPulseSamples) {
            if (d.ook_n <= 1) {
                d.st = kIdle;
                return 0;
            }
        } else {
            put(t.ook_pulse, d.ook_hw, d.ook_n, d.run);
            d.last_pulse = d.run;
            if (d.run > d.longest) d.longest = d.run;
            d.run = 0;
        }
        st = kGapStart;
    }
    if (st == kGapStart) {
        if (d.fsk_n > (unsigned)kMinPulses) {
            close_fsk(d, t, fpdm);
            return 2;
        }
    }
    put(t.ook_gap, d.ook_hw, d.ook_n, d.run);
    d.ook_n += 1;
    d.st = kIdle;
    return 1;
}

// Header of a finished package as the reference would leave it in pulse_data_t
struct PackageHeader {
    int type;
    unsigned num_pulses;
    unsigned long long offset;
    int low, high, f1, f2;
    unsigned long long start_abs;
};

R4_HD PackageHeader package_header(DetState const &d, int type)
{
    PackageHeader h;
    h.type = type;
    h.low = d.low;   // src/pulse_detect.c:247-248, :268-269, :395-396, :433-434, :455-456
    h.high = d.high;
    h.start_abs = d.start_abs;
    if (type == 1) {
        h.num_pulses = d.ook_n;
        h.offset = d.start_abs;
        h.f1 = d.ook_f1; // pulses->fsk_f1_est, tracked during pulses (:365); f2 stays 0
        h.f2 = 0;
    } else {
        h.num_pulses = d.fsk_n;
        h.offset = d.fsk_offset;
        h.f1 = d.fk_f1; // :393-394
        h.f2 = d.fk_f2;
    }
    return h;
}

// ------------------------------------------------------------- device counters --------

// The detector's words of a batch, zeroed in front of it: k_detect reserves packages and pool entries here, k_front
// and k_detect count what their shortcuts did (r433b_timing), k_mark reads the totals between pipelined launches
struct DetectCounters {
    unsigned pkgs, pool; // packages stored, pool entries reserved
    unsigned overflow;   // a package or its widths did not fit: the batch runs again with larger arenas
    unsigned unused;
    unsigned front_redone, front_repairs, idle_skipped, idle_rewalks, chain_folds, chain_fm_rebuilds;
};

// The slicers' words of a batch (k_slice2), zeroed in front of it
struct SliceCursor {
    unsigned long long bytes;    // event arena bytes reserved
    unsigned long long events;   // events stored
    unsigned long long overflow; // an output did not fit the arena: the batch slices again with a larger one
    unsigned long long gated;    // events dropped by a gate
};

static_assert(sizeof(DetectCounters) == 40 && sizeof(SliceCursor) == 32, "the counter buffers hold 64 bytes");

} // namespace r433b
