// r433b_split.cuh -- segmented replay (DESIGN §7c): the device side of the schedule that walks the segments of one long
// stream on separate warps.  k_front / k_detect walk the segments as chained chunks; the kernels here compare a segment's
// start state with its predecessor's end state, move start / end states between the slots, a rewalk launch and the
// slots of a chain, and merge the packages of every segment's last walk into the batch's arenas.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/r433b.h"
#include "r433b_detect.cuh"

namespace r433b {

constexpr int kSplitWarps = 4; // warps per CTA of the split kernels

// The scalar part of "the same future outputs from the same samples" (DESIGN §7c).  Left out: seq (renumbered by the
// merge), flushed (k_detect's first launch of a batch sets it to 0 before reading it), ook_hw / fsk_hw (they only say how
// far begin_package clears; the entries are compared instead, see split_trains_equal), last_start while last_count is 0
// (log_add overwrites it).  With the detector IDLE, the package fields are left out: begin_package sets every one of them
// (run, longest, ook_n, ook_f1, last_pulse, fsk_n, fsk_offset, start_abs, the FSK sub-detector) before it is read.
R4_HD bool split_scalar_equal(StreamState const &a, StreamState const &b)
{
    DetState const &x = a.d, &y = b.d;
    bool eq = x.st == y.st && x.lead_in == y.lead_in && x.low == y.low && x.high == y.high && x.eop_flag == y.eop_flag;
    eq = eq && a.y_am == b.y_am;
    eq = eq && a.fm_state.pos == b.fm_state.pos && a.fm_state.y == b.fm_state.y && a.fm_state.xf == b.fm_state.xf;
    eq = eq && a.fm_start.pos == b.fm_start.pos && a.fm_start.y == b.fm_start.y && a.fm_start.xf == b.fm_start.xf;
    eq = eq && a.iq_i == b.iq_i && a.iq_q == b.iq_q;
    eq = eq && a.log_n == b.log_n && a.last_count == b.last_count && (a.last_count == 0 || a.last_start == b.last_start);
    if (x.st != kIdle) {
        eq = eq && x.run == y.run && x.longest == y.longest && x.ook_n == y.ook_n && x.ook_f1 == y.ook_f1
                && x.last_pulse == y.last_pulse && x.fsk_n == y.fsk_n && x.fsk_offset == y.fsk_offset
                && x.start_abs == y.start_abs;
        eq = eq && x.fk_len == y.fk_len && x.fk_st == y.fk_st && x.fk_f1 == y.fk_f1 && x.fk_f2 == y.fk_f2
                && x.fk_vmax == y.fk_vmax && x.fk_vmin == y.fk_vmin && x.fk_skip == y.fk_skip;
    }
    return eq;
}

// The open package's train entries (one warp).  Entries at and behind a train's high-water mark are zero (begin_package
// clears [0, hw) and only put() raises hw; a fresh stream has hw = kMaxPulses), so comparing [0, max(hw_a, hw_b))
// compares the whole train.  With the detector IDLE the trains are not compared: begin_package clears them.
__device__ __forceinline__ bool split_trains_equal(StreamState const &a, StreamState const &b, int const *ta, int const *tb,
        int lane)
{
    unsigned const n_ook = a.d.ook_hw > b.d.ook_hw ? a.d.ook_hw : b.d.ook_hw;
    unsigned const n_fsk = a.d.fsk_hw > b.d.fsk_hw ? a.d.fsk_hw : b.d.fsk_hw;
    bool diff = false;
    for (unsigned i = (unsigned)lane; i < n_ook && i < (unsigned)kMaxPulses; i += 32)
        diff = diff || ta[i] != tb[i] || ta[kMaxPulses + i] != tb[kMaxPulses + i];
    for (unsigned i = (unsigned)lane; i < n_fsk && i < (unsigned)kMaxPulses; i += 32)
        diff = diff || ta[2 * kMaxPulses + i] != tb[2 * kMaxPulses + i] || ta[3 * kMaxPulses + i] != tb[3 * kMaxPulses + i];
    return __ballot_sync(0xffffffffu, diff) == 0;
}

// One warp per listed segment k: equal[i] = 1 when seed[k] (its start state) equals state[k - 1] (the end state of its
// predecessor's last walk), trains included.  start_seq[k] = the seed's seq, which pass 1 started segment k from.
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_compare(StreamState const *seed, int const *seed_train,
        StreamState const *state, int const *train, unsigned const *segs, unsigned n, unsigned char *equal,
        unsigned *start_seq)
{
    unsigned const i = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (i >= n) return;
    unsigned const k = segs[i];
    StreamState const a = seed[k], b = state[k - 1];
    bool eq = split_scalar_equal(a, b);
    if (eq && a.d.st != kIdle)
        eq = split_trains_equal(a, b, seed_train + (size_t)k * kTrainInts, train + (size_t)(k - 1) * kTrainInts, lane);
    if (lane == 0) {
        equal[i] = eq ? 1 : 0;
        start_seq[k] = a.seq;
    }
}

// R433B_SPOIL_SEED: perturb one value of every seed, cycling by segment index through the compared field groups, so that
// every seed is rejected (tests of the rewalk path)
__global__ void k_split_spoil(StreamState *seed, int *seed_train, unsigned n)
{
    unsigned const k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    StreamState &s = seed[k];
    int *const t = seed_train + (size_t)k * kTrainInts;
    bool const open = s.d.st != kIdle;
    switch (k % 9) {
    case 0: s.d.low ^= 1; break;
    case 1: s.d.lead_in += 1; break;
    case 2: s.y_am ^= 1; break;
    case 3: s.fm_state.y ^= 1; break;
    case 4: s.iq_i ^= 1; break;
    case 5: s.d.high ^= 1; break;
    case 6: // the carrier estimate of an open package, or the state itself
        if (open) s.d.ook_f1 ^= 1;
        else s.d.st = kGap;
        break;
    case 7: // the open package's trains
        if (open && s.d.ook_hw) t[0] ^= 1;
        else if (open && s.d.fsk_hw) t[2 * kMaxPulses] ^= 1;
        else s.d.eop_flag ^= 1;
        break;
    default: s.log_n += 1; break; // the deferred carrier-estimate log
    }
}

// One warp: the pulse trains of one slot (kTrainInts ints, 16-byte aligned) into another, in int4 words
__device__ __forceinline__ void split_copy_train(int const *src, int *dst, int lane)
{
    int4 const *s = reinterpret_cast<int4 const *>(src);
    int4 *d = reinterpret_cast<int4 *>(dst);
    for (int j = lane; j < kTrainInts / 4; j += 32) d[j] = s[j];
}

// One warp per listed segment k: the rewalk launch's stream i starts from the end state (and trains) of segment k - 1;
// start_seq[k] is the seq it starts from
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_gather(StreamState const *state, int const *train,
        unsigned const *segs, unsigned n, StreamState *rw_state, int *rw_train, unsigned *start_seq)
{
    unsigned const i = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (i >= n) return;
    unsigned const k = segs[i];
    split_copy_train(train + (size_t)(k - 1) * kTrainInts, rw_train + (size_t)i * kTrainInts, lane);
    if (lane == 0) {
        rw_state[i] = state[k - 1];
        start_seq[k] = state[k - 1].seq;
    }
}

// One warp per listed segment k: the end state of the rewalk launch's stream i becomes segment k's
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_scatter(StreamState const *rw_state, int const *rw_train,
        unsigned const *segs, unsigned n, StreamState *state, int *train)
{
    unsigned const i = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (i >= n) return;
    unsigned const k = segs[i];
    split_copy_train(rw_train + (size_t)i * kTrainInts, train + (size_t)k * kTrainInts, lane);
    if (lane == 0) state[k] = rw_state[i];
}

// Chained batches (r433b_chain_split), one warp per chain slot i whose file goes on (cont[i]): the slot's first segment
// first[i] starts from the state and trains the chain carried, and from its seq.  A slot that starts a file keeps the
// reset state pass 0 left in that segment's slot, and start_seq 0.
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_chain_in(StreamState const *chain_state,
        int const *chain_train, unsigned char const *cont, unsigned const *first, unsigned n, StreamState *state,
        int *train, unsigned *start_seq)
{
    unsigned const i = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (i >= n || !cont[i]) return;
    unsigned const k = first[i];
    split_copy_train(chain_train + (size_t)i * kTrainInts, train + (size_t)k * kTrainInts, lane);
    if (lane == 0) {
        state[k] = chain_state[i];
        start_seq[k] = chain_state[i].seq;
    }
}

// After the merge, one warp per chain slot i: the chain goes on from the end state and trains of the slot's last
// segment last[i].  That walk counted seq from its own start (a seed's counts the warm-up's packages), so the carried
// seq is the slot's start seq plus the packages merged for the slot.
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_chain_out(StreamState const *state, int const *train,
        unsigned const *first, unsigned const *last, unsigned const *start_seq, unsigned const *pkg_base, unsigned n,
        StreamState *chain_state, int *chain_train)
{
    unsigned const i = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (i >= n) return;
    unsigned const k = last[i], f = first[i];
    split_copy_train(train + (size_t)k * kTrainInts, chain_train + (size_t)i * kTrainInts, lane);
    if (lane == 0) {
        StreamState ss = state[k];
        ss.seq = start_seq[f] + pkg_base[k + 1] - pkg_base[f];
        chain_state[i] = ss;
    }
}

// What the merge reads per segment and per walk (host-built, except start_seq and pkg_base)
struct SplitMerge {
    unsigned n_segs, n_launches;
    unsigned const *seg_stream;  // the batch stream of segment k
    unsigned const *seg_first;   // the stream's first segment
    unsigned const *final_walk;  // the launch of segment k's last walk
    unsigned const *start_seq;   // the seq that walk started from
    StreamState const *state;    // ... and the state it ended in (its seq)
    unsigned const *launch_lo;   // n_launches + 1: launch l stored packages [launch_lo[l], launch_lo[l + 1])
    unsigned const *map_off;     // stream s of launch l walked segment seg_of[map_off[l] + s]
    unsigned const *seg_of;
    unsigned *pkg_base;          // n_segs + 1: merged position of segment k's first package; [n_segs] = the total
    r433b_package const *src;
    int const *src_pulse, *src_gap;
    r433b_package *dst;
    int *dst_pulse, *dst_gap;
    unsigned *pool_cursor;       // pool entries written
};

// One warp: pkg_base = exclusive prefix sum over the segments' package counts (end seq - start seq of the last walk)
__global__ void k_split_merge_scan(SplitMerge m)
{
    int const lane = threadIdx.x & 31;
    unsigned carry = 0;
    for (unsigned k0 = 0; k0 < m.n_segs; k0 += 32) {
        unsigned const k = k0 + (unsigned)lane;
        unsigned const c = k < m.n_segs ? m.state[k].seq - m.start_seq[k] : 0u;
        unsigned x = c;
        for (int d = 1; d < 32; d <<= 1) {
            unsigned const y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (k < m.n_segs) m.pkg_base[k] = carry + x - c;
        carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) m.pkg_base[m.n_segs] = carry;
}

// One warp per stored package: a package of its segment's last walk goes to pkg_base[seg] + (seq - start_seq) with the
// batch's stream, the seq the one-warp walk gives it and its widths copied to the next free pool entries.  The seq goes
// on from the stream's first segment's start seq: 0, or what a chained batch's slot carried.
__global__ void __launch_bounds__(kSplitWarps * 32) k_split_merge(SplitMerge m)
{
    unsigned const idx = blockIdx.x * kSplitWarps + (threadIdx.x >> 5);
    int const lane = threadIdx.x & 31;
    if (idx >= m.launch_lo[m.n_launches]) return;
    unsigned lo = 0, hi = m.n_launches; // the launch l with launch_lo[l] <= idx < launch_lo[l + 1]
    while (hi - lo > 1) {
        unsigned const mid = (lo + hi) / 2;
        if (m.launch_lo[mid] <= idx) lo = mid;
        else hi = mid;
    }
    r433b_package k = m.src[idx];
    unsigned const seg = m.seg_of[m.map_off[lo] + k.stream];
    if (m.final_walk[seg] != lo) return;
    unsigned const rel = k.seq - m.start_seq[seg];
    unsigned off = 0;
    if (lane == 0) off = atomicAdd(m.pool_cursor, k.pulse_count);
    off = __shfl_sync(0xffffffffu, off, 0);
    for (unsigned j = (unsigned)lane; j < k.pulse_count; j += 32) {
        m.dst_pulse[off + j] = m.src_pulse[k.pulse_off + j];
        m.dst_gap[off + j] = m.src_gap[k.pulse_off + j];
    }
    if (lane == 0) {
        k.stream = m.seg_stream[seg];
        unsigned const first = m.seg_first[seg];
        k.seq = m.start_seq[first] + m.pkg_base[seg] - m.pkg_base[first] + rel;
        k.pulse_off = off;
        m.dst[m.pkg_base[seg] + rel] = k;
    }
}

} // namespace r433b
