// r433b_mixed.cuh -- mixed batches (r433b_process_mixed, DESIGN §7d): k_mixed_order puts the packages of the concurrent
// class launches back in order.  The launches append to one package arena in completion order, interleaved; k_slice2
// needs one contiguous package range per sample rate.  Three passes of the same kernel: count the packages of every
// internal stream, scan the counts in internal order (streams sorted by class, so every rate slot is one run of them),
// scatter every header to base[stream] + seq - start_seq[stream] with the caller's stream index.  A stream's packages of
// one batch have seq start_seq .. start_seq + count - 1 (start_seq: 0, or the seq a chain slot carried in), so the order
// is (internal stream, seq) whatever order the launches stored them in.  The widths stay in the pools (pulse_off is
// kept).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/r433b.h"

namespace r433b {

constexpr int kMixedThreads = 256;

struct MixedOrder {
    r433b_package const *src; // n_pkgs headers as the detector stored them (stream = internal index)
    r433b_package *dst;       // the same headers grouped by rate slot
    unsigned n_pkgs;
    unsigned n_streams;       // internal streams
    unsigned const *caller;   // caller's index of internal stream s
    unsigned *base;           // n_streams + 1: packages per stream (pass 0), then their first position (pass 1)
    unsigned const *start_seq; // seq of internal stream s's first package of the batch; nullptr: 0 (unchained)
};

// pass 0: count (grid-stride, base zeroed by the host); pass 1: exclusive scan in place (one warp); pass 2: scatter
__global__ void __launch_bounds__(kMixedThreads) k_mixed_order(MixedOrder m, int pass)
{
    if (pass == 1) {
        int const lane = threadIdx.x & 31;
        if (threadIdx.x >= 32) return;
        unsigned carry = 0;
        for (unsigned s0 = 0; s0 < m.n_streams; s0 += 32) {
            unsigned const s = s0 + (unsigned)lane;
            unsigned const c = s < m.n_streams ? m.base[s] : 0u;
            unsigned x = c;
            for (int d = 1; d < 32; d <<= 1) {
                unsigned const y = __shfl_up_sync(0xffffffffu, x, d);
                if (lane >= d) x += y;
            }
            if (s < m.n_streams) m.base[s] = carry + x - c;
            carry += __shfl_sync(0xffffffffu, x, 31);
        }
        if (lane == 0) m.base[m.n_streams] = carry;
        return;
    }
    for (unsigned i = blockIdx.x * kMixedThreads + threadIdx.x; i < m.n_pkgs; i += gridDim.x * kMixedThreads) {
        if (pass == 0) {
            atomicAdd(&m.base[m.src[i].stream], 1u);
        } else {
            r433b_package k = m.src[i];
            unsigned const at = m.base[k.stream] + k.seq - (m.start_seq ? m.start_seq[k.stream] : 0u);
            k.stream = m.caller[k.stream];
            m.dst[at] = k;
        }
    }
}

} // namespace r433b
