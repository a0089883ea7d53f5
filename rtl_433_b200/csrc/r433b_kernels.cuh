// r433b_kernels.cuh -- the other sm_90a kernels of the IQ -> package -> event path:
//
//   k_detect (r433b_detect.cuh) : one WARP per capture stream, IQ -> packages.
//   k_cf32_to_cs16              : float IQ captures to cs16 in front of k_detect.
//   k_bucket_count/scan/scatter : the packages of a range sorted by (type, length) for k_slice2, and their widths
//                                 copied lane-interleaved.
//   k_slice2                    : one thread per (package, device), a warp = 32 packages of one device: every pulse
//                                 slicer on every package, events staged per thread and copied into the arena by the warp.
//   k_mark                      : one-thread bookkeeping between the launches of a pipelined batch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/r433b.h"
#include "r433b_core.cuh"
#include "r433b_slice.cuh"
#include "r433b_detect.cuh"

namespace r433b {

// ----------------------------------------------------------------- cf32 -> cs16 ----------

// src/rtl_433.c:1811-1825: "clamp float to [-1,1] and scale to Q0.15" -- the reference converts a
// cf32 capture to cs16 before anything else looks at it.  Streaming, HBM bound (12 B per float pair
// of traffic per 2 samples); `n4` groups of four floats.  The out-of-range / NaN case follows the
// reference's x86-64 builds: the conversion yields INT_MIN, the clamp makes it -32767.
__global__ void k_cf32_to_cs16(float4 const *in, uint2 *out, size_t n4)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 v = __ldcs(in + i);
        float f[4] = {v.x, v.y, v.z, v.w};
        int s[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float t = __fmul_rn(f[k], 32767.0f);
            int q = (t >= -2147483648.0f && t < 2147483648.0f) ? __float2int_rz(t) : (int)0x80000000;
            q = q < -32767 ? -32767 : (q > 32767 ? 32767 : q);
            s[k] = q;
        }
        uint2 o;
        o.x = (uint32_t)(uint16_t)(int16_t)s[0] | ((uint32_t)(uint16_t)(int16_t)s[1] << 16);
        o.y = (uint32_t)(uint16_t)(int16_t)s[2] | ((uint32_t)(uint16_t)(int16_t)s[3] << 16);
        out[i] = o;
    }
}

// ------------------------------------------------------------------------- k_slice2 ------

// What one pipeline group (a contiguous run of streams) produced, filled on the device so the
// next stage never waits for the host.
struct GroupRange {
    unsigned pkg_begin, pkg_end;
    unsigned pool_begin, pool_end;
    unsigned long long arena_begin, arena_end;
    unsigned long long events_end, gated_end;
    unsigned overflow; // bit 0: the detector's arenas, bit 1: the event arena, bit 2: k_slice2's width copy
    unsigned next; // k_slice2 work counter: next (device, package group) item of this range
    // k_bucket: the packages of the range sorted by type, then by descending num_pulses, in `order[pkg_begin + ...]`:
    // count[0] OOK packages, then count[1] FSK ones, in groups[t] groups of 32 per type
    unsigned count[2], groups[2];
};

__global__ void k_mark(GroupRange *r, int which, DetectCounters const *counters, SliceCursor const *cursor)
{
    if (which == 0) {
        r->pkg_begin = counters->pkgs;
        r->pool_begin = counters->pool;
    } else if (which == 1) {
        r->pkg_end = counters->pkgs;
        r->pool_end = counters->pool;
        r->overflow = counters->overflow;
        r->next = 0;
    } else if (which == 2) {
        r->arena_begin = cursor->bytes;
    } else {
        r->arena_end = cursor->bytes;
        r->events_end = cursor->events;
        r->gated_end = cursor->gated;
        r->overflow |= (unsigned)cursor->overflow << 1;
    }
}

// The 32 lanes of a k_slice2 warp are 32 PACKAGES looked at by ONE device.  Lanes that were 32 devices on one
// package would interpret the same pulse with 32 different sets of limits and so want 32 different things from the
// bit writer; here all lanes carry the same limits, walk packages of the same type and length (k_bucket), and pulse
// n of one burst is the same kind of thing as pulse n of another -- the lanes differ in data (which bit), far less
// in control flow.  A warp runs until its longest lane is done, so its 32 packages are 32 consecutive ones of the
// range sorted by length.
//
// k_bucket also gives k_slice2 its own copy of the widths, lane-interleaved per group: row k (pulse k and the gap
// after it) of the package in lane l of group g is copy[base[g] + 32 k + l], so that one step of a warp is one
// coalesced 256-byte load instead of 64 lines, and the rows of a group are as many as its first (longest) package has
// entries.  Rows past a shorter package's own entries are padding that no slicer reads.  Groups are sorted by
// descending length, so group g + 1 has no more rows than any package of the full group g before it: the copy of a
// type takes at most its pool entries plus 32 x kMaxPulses.
constexpr unsigned kLenBins = kMaxPulses + 1; // num_pulses 0 .. kMaxPulses

// num_pulses as a histogram bin (a record that is not a package of this batch -- the stale ones a detector overflow
// leaves in a range that is redone -- must stay inside the tables), and the rows it takes in the copy: the package's
// pool entries (r433b_package.pulse_count), where the entry after the last pulse is part of the record
__host__ __device__ inline unsigned len_bin(unsigned num_pulses) { return num_pulses < kLenBins ? num_pulses : kMaxPulses; }
__host__ __device__ inline unsigned copy_rows(unsigned len) { return len < (unsigned)kMaxPulses ? len + 1 : kMaxPulses; }

struct SortScratch {
    unsigned *hist;     // 2 x kLenBins: packages per (type, length); zero between ranges (k_bucket_scan clears it)
    unsigned *fill;     // 2 x kLenBins: k_bucket_scatter's next position per (type, length)
    unsigned *base;     // per group, OOK ones first, and one past the last: its first entry in `copy`
    PulseGap *copy;
    unsigned long long copy_cap; // entries
};

// Sort the packages of a range into order[pkg_begin ...) and fill the copy: count, scan, scatter -- three small
// launches without a block barrier (grid-stride loops; the range is only known on the device).  The count pass also
// gives every package its row in the pair table.
constexpr int kBucketThreads = 256;
__global__ void __launch_bounds__(kBucketThreads) k_bucket_count(GroupRange *r, r433b_package *pkgs, unsigned n_pkgs, unsigned n_devs, unsigned *hist)
{
    unsigned const b0 = r->pkg_begin, b1 = r->pkg_end < n_pkgs ? r->pkg_end : n_pkgs;
    for (unsigned pk = b0 + blockIdx.x * kBucketThreads + threadIdx.x; pk < b1; pk += gridDim.x * kBucketThreads) {
        r433b_package const k = pkgs[pk];
        pkgs[pk].first_pair = pk * n_devs;
        atomicAdd(&hist[(k.type == 1 ? 0 : kLenBins) + len_bin(k.num_pulses)], 1u);
    }
}

// One warp, on a copy of the histogram in shared memory.  The bins in sorted order (OOK, then FSK; longest first)
// give every bin its first position; every group of 32 positions takes as many rows as the bin of its first one, and a
// prefix over the bins of the groups starting in them places the groups in the copy.
__global__ void __launch_bounds__(32) k_bucket_scan(GroupRange *r, SortScratch s)
{
    constexpr unsigned kBins = 2 * kLenBins, kPer = (kBins + 31) / 32; // consecutive bins of the sorted order per lane
    __shared__ unsigned hist[kPer * 32];
    unsigned const lane = threadIdx.x;
    auto len = [](unsigned i) { return i < kLenBins ? kMaxPulses - i : kLenBins + kMaxPulses - i; }; // i: sorted order
    for (unsigned i = lane; i < kPer * 32; i += 32) hist[i] = i < kBins ? s.hist[(i < kLenBins ? 0 : kLenBins) + len(i)] : 0;
    __syncwarp();
    unsigned n0 = 0, n1 = 0;
    for (unsigned j = 0; j < kPer; ++j) {
        unsigned const i = lane * kPer + j;
        (i < kLenBins ? n0 : n1) += hist[i];
    }
    unsigned at = n0 + n1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned const v = __shfl_up_sync(0xffffffffu, at, o);
        if ((int)lane >= o) at += v;
    }
    at -= n0 + n1; // first position of the lane's first bin
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        n0 += __shfl_xor_sync(0xffffffffu, n0, o);
        n1 += __shfl_xor_sync(0xffffffffu, n1, o);
    }
    unsigned const g0 = (n0 + 31) / 32, g1 = (n1 + 31) / 32;
    // the copy entries of the groups whose first position lies in the lane's bins
    unsigned long long e = 0;
    for (unsigned j = 0, a = at; j < kPer; ++j) {
        unsigned const i = lane * kPer + j, n = hist[i];
        unsigned const q = a - (i < kLenBins ? 0 : n0); // within the type
        e += (unsigned long long)((q + n + 31) / 32 - (q + 31) / 32) * 32 * copy_rows(len(i));
        a += n;
    }
    unsigned long long incl = e;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned long long const v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += v;
    }
    unsigned long long const total = __shfl_sync(0xffffffffu, incl, 31);
    // only records that are not this batch's packages (a detector overflow, whose range is redone) can outgrow the
    // copy: the range then slices nothing
    bool const fits = total <= s.copy_cap;
    e = incl - e;
    for (unsigned j = 0; j < kPer; ++j) {
        unsigned const i = lane * kPer + j, n = hist[i];
        if (i >= kBins) break;
        unsigned const t = i < kLenBins ? 0 : 1, b = t * kLenBins + len(i), q = at - (t ? n0 : 0);
        s.fill[b] = at;
        if (n) s.hist[b] = 0;
        unsigned const size = 32 * copy_rows(len(i));
        for (unsigned g = (q + 31) / 32; g * 32 < q + n; ++g, e += size) s.base[(t ? g0 : 0) + g] = (unsigned)e;
        at += n;
    }
    if (lane == 0) {
        s.base[g0 + g1] = (unsigned)total;
        r->count[0] = n0;
        r->count[1] = n1;
        r->groups[0] = fits ? g0 : 0;
        r->groups[1] = fits ? g1 : 0;
        if (!fits) r->overflow |= 4;
        r->next = 0;
    }
}

// Every package to its sorted position, and its rows into the copy.  The warp copies its 32 packages one after the
// other, 32 rows at a time, so that the pool reads are whole lines.
__global__ void __launch_bounds__(kBucketThreads) k_bucket_scatter(GroupRange *r, r433b_package const *pkgs, unsigned n_pkgs, unsigned *order,
                                                                  SortScratch s, int const *pulse_pool, int const *gap_pool)
{
    unsigned const lane = threadIdx.x & 31;
    unsigned const b0 = r->pkg_begin, b1 = r->pkg_end < n_pkgs ? r->pkg_end : n_pkgs;
    unsigned const n0 = r->count[0], g0 = r->groups[0], g1 = r->groups[1];
    for (unsigned w = b0 + blockIdx.x * kBucketThreads + threadIdx.x - lane; w < b1; w += gridDim.x * kBucketThreads) {
        unsigned const pk = w + lane;
        unsigned dst = 0, rows = 0, off = 0;
        if (pk < b1) {
            r433b_package const k = pkgs[pk];
            unsigned const t = k.type == 1 ? 0 : 1, len = len_bin(k.num_pulses);
            unsigned const pos = atomicAdd(&s.fill[t * kLenBins + len], 1u);
            order[b0 + pos] = pk;
            unsigned const q = pos - (t ? n0 : 0);
            if (q / 32 < (t ? g1 : g0)) {
                dst = s.base[(t ? g0 : 0) + q / 32] + q % 32;
                rows = copy_rows(len);
                off = k.pulse_off;
            }
        }
        for (int l = 0; l < 32; ++l) {
            unsigned const n = __shfl_sync(0xffffffffu, rows, l), d = __shfl_sync(0xffffffffu, dst, l);
            unsigned const o = __shfl_sync(0xffffffffu, off, l);
            for (unsigned k = lane; k < n; k += 32) s.copy[d + 32 * k] = PulseGap{pulse_pool[o + k], gap_pool[o + k]};
        }
    }
}

struct SliceParams {
    r433b_package const *pkgs;
    GroupRange *range; // the packages of the range (k_bucket's counts) and the work counter
    unsigned const *order; // k_bucket's output
    PulseGap const *copy;  // k_bucket's lane-interleaved widths
    unsigned const *group_base;
    SlicerParams const *dev;  // per device, already scaled to the sample rate of the range
    unsigned n_devs;
    unsigned const *ook_list, *fsk_list; // device indices taking OOK / FSK packages, grouped by modulation
    unsigned n_ook, n_fsk;
    r433b_pair *pairs;        // n_pkgs * n_devs, pre-zeroed
    uint8_t *arena;
    unsigned long long arena_cap;
    SliceCursor *cursor;
    uint32_t *stage;          // kStageWords per thread of the (fixed) grid
};

constexpr int kSliceThreads = 128;
constexpr unsigned kStageWords = 1024; // scratch words per k_slice2 thread (4 KiB): larger outputs take the second pass
constexpr int kSliceCtasPerSm = 8; // 64 registers, 32 warps/SM.  Gated, 4096 x 2^20 cu8: 6 CTAs/SM 7.0 ms, 8 -> 6.3,
                                   // 12 -> 9.9 (40 registers spill)

// k_slice2's shared memory: the threads' write-combining windows, a column each (a lane always hits its own bank),
// and per thread the first word of its output in the warp's arena range and the first one still in its window
__shared__ uint32_t g_slice_win[kSliceWindow][kSliceThreads];
__shared__ unsigned g_slice_seg[2][kSliceThreads];
struct SliceWindow {
    static constexpr bool kOn = true;
    __device__ __forceinline__ static uint32_t &slot(unsigned s) { return g_slice_win[s][threadIdx.x]; }
};

// One slicing pass per (package, device) item: the events go through the thread's window into its scratch, and the
// warp copies the outputs of its 32 lanes, which are one contiguous arena range, in whole lines.  A warp with a lane
// whose output outgrows the scratch slices again, straight into the arena.
__global__ void __launch_bounds__(kSliceThreads, kSliceCtasPerSm) k_slice2(SliceParams p)
{
    unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    GroupRange const *rg = p.range;
    unsigned const pk_begin = rg->pkg_begin;
    unsigned const groups_ook = rg->groups[0], groups_fsk = rg->groups[1];
    // items: device major (at any moment most warps of the GPU run the same device, so the same code), OOK devices
    // on the OOK packages first
    unsigned const items_ook = p.n_ook * groups_ook, items = items_ook + p.n_fsk * groups_fsk;
    uint32_t *stage = p.stage + ((size_t)blockIdx.x * kSliceThreads + threadIdx.x) * kStageWords;
    for (;;) {
        unsigned item = 0;
        if (lane == 0) item = atomicAdd(&p.range->next, 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= items) break;
        int const t = item < items_ook ? 0 : 1;
        unsigned const rel = t ? item - items_ook : item;
        unsigned const groups = t ? groups_fsk : groups_ook;
        unsigned const slot = rel / groups;
        unsigned const g = rel - slot * groups;
        unsigned const dev = (t ? p.fsk_list : p.ook_list)[slot];
        unsigned const in_type = g * 32 + lane;
        bool const active = in_type < rg->count[t];
        unsigned const pk = active ? p.order[pk_begin + (t ? rg->count[0] : 0) + in_type] : 0;
        SlicerParams const sp = p.dev[dev];
        PulseViewT<32> pv;
        pv.w = p.copy + p.group_base[(t ? groups_ook : 0) + g] + lane;
        pv.n = active ? len_bin(p.pkgs[pk].num_pulses) : 0;
        unsigned bytes = 0, nev = 0, ng1 = 0, ngN = 0, wb = 0;
        if (active) {
            EventWriterT<SliceWindow> w;
            w.init(stage, kStageWords, (unsigned)sp.gate);
            slice_dispatch(pv, sp, w);
            bytes = w.committed * 4;
            wb = w.wb;
            nev = w.events;
            ng1 = w.gated1;
            ngN = w.gatedN;
        }
        unsigned incl = bytes;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += v;
        }
        unsigned const total = __shfl_sync(0xffffffffu, incl, 31);
        unsigned evs = nev, dropped = ng1 + ngN;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            evs += __shfl_xor_sync(0xffffffffu, evs, o);
            dropped += __shfl_xor_sync(0xffffffffu, dropped, o);
        }
        unsigned long long wbase = 0;
        if (lane == 0 && total) {
            wbase = atomicAdd(&p.cursor->bytes, (unsigned long long)total);
            atomicAdd(&p.cursor->events, (unsigned long long)evs);
        }
        if (lane == 0 && dropped) atomicAdd(&p.cursor->gated, (unsigned long long)dropped);
        wbase = __shfl_sync(0xffffffffu, wbase, 0);
        unsigned long long const off = wbase + incl - bytes;
        bool const fits = off + bytes <= p.arena_cap;
        if (active && bytes && !fits) atomicOr(&p.cursor->overflow, 1ull);
        if (__all_sync(0xffffffffu, bytes <= kStageWords * 4)) {
            // word i of the warp's range [wbase, wbase + total) belongs to the last lane whose output starts at or
            // before i; the lanes take 32 consecutive words, aligned to a 128-byte line, at a time
            unsigned const first = (incl - bytes) / 4;
            g_slice_seg[0][threadIdx.x] = first;
            g_slice_seg[1][threadIdx.x] = first + wb;
            __syncwarp();
            unsigned const w0 = threadIdx.x - lane;
            unsigned n = total / 4; // the words that fit in the arena (a lane that does not fit is redone)
            if (wbase + total > p.arena_cap) n = wbase >= p.arena_cap ? 0 : (unsigned)((p.arena_cap - wbase) / 4);
            unsigned const lead = (unsigned)(wbase / 4) & 31;
            uint32_t *to = reinterpret_cast<uint32_t *>(p.arena + wbase) - lead;
            uint32_t const *scratch = stage - (size_t)lane * kStageWords; // lane 0's
            for (unsigned j = lane; j < n + lead; j += 32) {
                if (j < lead) continue;
                unsigned const i = j - lead;
                unsigned l = 0;
#pragma unroll
                for (unsigned s = 16; s; s >>= 1)
                    if (g_slice_seg[0][w0 + l + s] <= i) l += s;
                unsigned const at = i - g_slice_seg[0][w0 + l];
                uint32_t const v = i >= g_slice_seg[1][w0 + l] ? g_slice_win[at % kSliceWindow][w0 + l]
                                                               : scratch[(size_t)l * kStageWords + at];
                __stcs(to + j, v);
            }
            __syncwarp();
        } else if (active && bytes && fits) {
            EventWriter w;
            w.init(reinterpret_cast<uint32_t *>(p.arena + off), bytes / 4, (unsigned)sp.gate);
            slice_dispatch(pv, sp, w);
        }
        if (active) {
            r433b_pair pr;
            pr.offset = off;
            pr.bytes = bytes;
            pr.events = nev;
            pr.gated_single = ng1;
            pr.gated_multi = ngN;
            p.pairs[(size_t)pk * p.n_devs + dev] = pr;
        }
    }
}

} // namespace r433b
