// r433b_kernels.cuh -- the other sm_90a kernels of the IQ -> package -> event path:
//
//   k_detect (r433b_detect.cuh) : one WARP per capture stream, IQ -> packages.
//   k_cf32_to_cs16              : float IQ captures to cs16 in front of k_detect.
//   k_bucket_count/scan/scatter : the packages of a range sorted by (type, length class) for k_slice2.
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

constexpr int kLenBuckets = 4; // length classes of packages: < 64, < 160, < 400 pulses, longer
__host__ __device__ inline int len_bucket(unsigned num_pulses)
{
    return num_pulses < 64 ? 0 : num_pulses < 160 ? 1 : num_pulses < 400 ? 2 : 3;
}

// What one pipeline group (a contiguous run of streams) produced, filled on the device so the
// next stage never waits for the host.
struct GroupRange {
    unsigned pkg_begin, pkg_end;
    unsigned pool_begin, pool_end;
    unsigned long long arena_begin, arena_end;
    unsigned long long events_end, gated_end;
    unsigned overflow;
    unsigned next; // k_slice2 work counter: next (device, package group) item of this range
    // k_bucket: the packages of the range sorted by (type, length class) in `order[pkg_begin + ...]`
    unsigned seg_begin[2][kLenBuckets], seg_count[2][kLenBuckets], seg_fill[2][kLenBuckets];
    unsigned groups[2]; // per type: sum over the buckets of ceil(count / 32)
};

__global__ void k_mark(GroupRange *r, int which, unsigned const *counters, unsigned long long const *cursor)
{
    if (which == 0) {
        r->pkg_begin = counters[0];
        r->pool_begin = counters[1];
    } else if (which == 1) {
        r->pkg_end = counters[0];
        r->pool_end = counters[1];
        r->overflow = counters[2];
        r->next = 0;
        for (int i = 0; i < 2 * kLenBuckets; ++i) (&r->seg_count[0][0])[i] = 0;
    } else if (which == 2) {
        r->arena_begin = cursor[0];
    } else {
        r->arena_end = cursor[0];
        r->events_end = cursor[1];
        r->gated_end = cursor[3];
        r->overflow |= (unsigned)cursor[2] << 1;
    }
}

// The 32 lanes of a k_slice2 warp are 32 PACKAGES looked at by ONE device.  Lanes that were 32 devices on one
// package would interpret the same pulse with 32 different sets of limits and so want 32 different things from the
// bit writer; here all lanes carry the same limits, walk packages of the same type and similar length (k_bucket), and
// pulse n of one burst is the same kind of thing as pulse n of another -- the lanes differ in data (which bit), far
// less in control flow.

// Sort the packages of a range by (type, length class) into order[pkg_begin ...): count, scan, scatter -- three small
// launches without a block barrier (grid-stride loops; the range is only known on the device).  The count pass also
// gives every package its row in the pair table.
constexpr int kBucketThreads = 256;
__global__ void __launch_bounds__(kBucketThreads) k_bucket_count(GroupRange *r, r433b_package *pkgs, unsigned n_pkgs, unsigned n_devs)
{
    unsigned const b0 = r->pkg_begin, b1 = r->pkg_end < n_pkgs ? r->pkg_end : n_pkgs;
    for (unsigned pk = b0 + blockIdx.x * kBucketThreads + threadIdx.x; pk < b1; pk += gridDim.x * kBucketThreads) {
        r433b_package const k = pkgs[pk];
        pkgs[pk].first_pair = pk * n_devs;
        atomicAdd(&r->seg_count[k.type == 1 ? 0 : 1][len_bucket(k.num_pulses)], 1u);
    }
}

__global__ void k_bucket_scan(GroupRange *r)
{
    unsigned at = 0;
    for (int t = 0; t < 2; ++t) {
        unsigned g = 0;
        for (int b = 0; b < kLenBuckets; ++b) {
            r->seg_begin[t][b] = at;
            r->seg_fill[t][b] = 0;
            at += r->seg_count[t][b];
            g += (r->seg_count[t][b] + 31) / 32;
        }
        r->groups[t] = g;
    }
    r->next = 0;
}

__global__ void __launch_bounds__(kBucketThreads) k_bucket_scatter(GroupRange *r, r433b_package const *pkgs, unsigned n_pkgs, unsigned *order)
{
    unsigned const b0 = r->pkg_begin, b1 = r->pkg_end < n_pkgs ? r->pkg_end : n_pkgs;
    for (unsigned pk = b0 + blockIdx.x * kBucketThreads + threadIdx.x; pk < b1; pk += gridDim.x * kBucketThreads) {
        r433b_package const k = pkgs[pk];
        int const t = k.type == 1 ? 0 : 1, b = len_bucket(k.num_pulses);
        unsigned const pos = r->seg_begin[t][b] + atomicAdd(&r->seg_fill[t][b], 1u);
        order[b0 + pos] = pk;
    }
}

struct SliceParams {
    r433b_package const *pkgs;
    GroupRange *range; // the packages of the range (k_bucket's segments) and the work counter
    unsigned const *order; // k_bucket's output
    int const *pulse_pool, *gap_pool;
    SlicerParams const *dev;  // per device, already scaled to the sample rate of the range
    unsigned n_devs;
    unsigned const *ook_list, *fsk_list; // device indices taking OOK / FSK packages, grouped by modulation
    unsigned n_ook, n_fsk;
    r433b_pair *pairs;        // n_pkgs * n_devs, pre-zeroed
    uint8_t *arena;
    unsigned long long arena_cap;
    unsigned long long *cursor; // [0] bytes reserved, [1] events stored, [2] overflow, [3] events dropped by a gate
    uint32_t *stage;            // kStageWords per thread of the (fixed) grid
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
        unsigned g = rel - slot * groups;
        unsigned const dev = (t ? p.fsk_list : p.ook_list)[slot];
        int b = 0;
        for (; b < kLenBuckets - 1; ++b) {
            unsigned const gb = (rg->seg_count[t][b] + 31) / 32;
            if (g < gb) break;
            g -= gb;
        }
        unsigned const in_seg = g * 32 + lane;
        bool const active = in_seg < rg->seg_count[t][b];
        unsigned const pk = active ? p.order[pk_begin + rg->seg_begin[t][b] + in_seg] : 0;
        SlicerParams const sp = p.dev[dev];
        PulseView pv;
        pv.pulse = p.pulse_pool;
        pv.gap = p.gap_pool;
        pv.n = 0;
        if (active) {
            r433b_package const k = p.pkgs[pk];
            pv.pulse = p.pulse_pool + k.pulse_off;
            pv.gap = p.gap_pool + k.pulse_off;
            pv.n = k.num_pulses;
        }
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
            wbase = atomicAdd(p.cursor, (unsigned long long)total);
            atomicAdd(p.cursor + 1, (unsigned long long)evs);
        }
        if (lane == 0 && dropped) atomicAdd(p.cursor + 3, (unsigned long long)dropped);
        wbase = __shfl_sync(0xffffffffu, wbase, 0);
        unsigned long long const off = wbase + incl - bytes;
        bool const fits = off + bytes <= p.arena_cap;
        if (active && bytes && !fits) atomicOr(p.cursor + 2, 1ull);
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
