// r433b_grab.cuh -- k_grab: the signal grabber's gather (src/samp_grab.c:98-170).  The windows of a grab plan are
// written back to back into a staging buffer, which then goes to the host in one copy.  The host cuts every window
// into segments: a run of bytes of the batch as it lies on the device (streams skip the padding between them),
// of the device copy of the previous batch's ring tail, or zeros (ring bytes the run never wrote).  Segments start on
// sample boundaries (2 or 4 bytes), so a source is read with aligned 16-byte loads and shifted into place; the word a
// lane needs behind its own comes from the next lane.  Each warp stores whole 512-byte spans (four 128-byte lines).
// One pass over the bytes: the bound is HBM, 2 x the bytes gathered.
//
// On a grabbing chain (r433b_chain_grab) every slot is its own run with its own ring on the device.  k_grab_ring
// appends each slot's chunk to its ring after the batch, and a chained plan's windows read the ring (kGrabRing,
// segments split at the ring's wrap by the host), the chunk where the ring no longer holds it (kGrabBatch), and the
// older ring bytes the append overwrote that the call's frames still need (kGrabPrior, saved by k_grab from the ring).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace r433b {

struct GrabSeg {
    unsigned long long dst; // first staging byte
    unsigned long long src; // byte offset into the source; kGrabRing: the ring byte's device address
    unsigned long long len;
    unsigned kind;          // kGrabZero / kGrabBatch / kGrabPrior / kGrabRing
    unsigned pad_;
};
enum : unsigned { kGrabZero = 0, kGrabBatch = 1, kGrabPrior = 2, kGrabRing = 3 };

struct GrabParams {
    uint8_t const *batch;   // 16-byte aligned
    uint8_t const *prior;   // 16-byte aligned
    GrabSeg const *segs;    // sorted by dst, covering [0, total) without gaps
    unsigned n_segs;
    unsigned flip;          // XORed into batch bytes: 0x80808080 turns cs8 into cu8
    unsigned long long total;
    uint4 *out;             // staging, total rounded up to kGrabSpan
};

constexpr int kGrabThreads = 256;
constexpr unsigned kGrabLine = 512;                        // bytes a warp stores per step: 32 lanes x 16
constexpr unsigned kGrabSteps = 16;                        // steps per warp
constexpr unsigned long long kGrabSpan = (unsigned long long)kGrabLine * kGrabSteps;
constexpr unsigned kGrabRingBytes = 12u * 262144u;         // R433B_GRAB_RING, a multiple of 16

// bytes [m, m + 16) of the 32 bytes a || b
__device__ __forceinline__ uint4 grab_shift(uint4 a, uint4 b, unsigned m)
{
    if (m & 8) {
        a.x = a.z, a.y = a.w, a.z = b.x, a.w = b.y;
        b.x = b.z, b.y = b.w;
    }
    if (m & 4) {
        a.x = a.y, a.y = a.z, a.z = a.w, a.w = b.x;
        b.x = b.y;
    }
    unsigned const k = m & 3;
    if (k) {
        unsigned const sel = k | (k + 1) << 4 | (k + 2) << 8 | (k + 3) << 12;
        a.x = __byte_perm(a.x, a.y, sel);
        a.y = __byte_perm(a.y, a.z, sel);
        a.z = __byte_perm(a.z, a.w, sel);
        a.w = __byte_perm(a.w, b.x, sel);
    }
    return a;
}

__global__ void __launch_bounds__(kGrabThreads) k_grab(GrabParams p)
{
    unsigned const lane = threadIdx.x & 31;
    unsigned long long const warp = ((unsigned long long)blockIdx.x * kGrabThreads + threadIdx.x) >> 5;
    unsigned long long const base = warp * kGrabSpan;
    if (base >= p.total) return; // warp-uniform
    // the segment holding this lane's first byte; later steps advance it
    unsigned long long d = base + lane * 16u;
    unsigned s = 0;
    {
        unsigned lo = 0, hi = p.n_segs;
        while (hi - lo > 1) {
            unsigned const mid = (lo + hi) >> 1;
            if (p.segs[mid].dst <= d) lo = mid;
            else hi = mid;
        }
        s = lo;
    }
    for (unsigned step = 0; step < kGrabSteps; ++step, d += kGrabLine) {
        if (base + step * kGrabLine >= p.total) break; // warp-uniform
        while (s + 1 < p.n_segs && p.segs[s + 1].dst <= d) ++s;
        GrabSeg const g = p.segs[s];
        // fast path: the lane's 16 bytes lie in one segment
        bool const whole = d < p.total && d + 16 <= g.dst + g.len;
        unsigned long long const src = g.kind == kGrabBatch ? (unsigned long long)p.batch
                                     : g.kind == kGrabPrior ? (unsigned long long)p.prior : 0ull;
        unsigned long long const at = g.src + (d - g.dst);
        bool const loads = whole && g.kind != kGrabZero;
        uint4 a = {0u, 0u, 0u, 0u};
        if (loads) a = __ldcs((uint4 const *)(src + (at & ~15ull)));
        // the aligned word behind this lane's is the next lane's own when both read the same source in order
        unsigned long long const key = loads ? src + (at & ~15ull) : 0ull;
        unsigned long long const next_key = __shfl_down_sync(0xffffffffu, key, 1);
        uint4 b;
        b.x = __shfl_down_sync(0xffffffffu, a.x, 1);
        b.y = __shfl_down_sync(0xffffffffu, a.y, 1);
        b.z = __shfl_down_sync(0xffffffffu, a.z, 1);
        b.w = __shfl_down_sync(0xffffffffu, a.w, 1);
        uint4 v = {0u, 0u, 0u, 0u};
        if (loads) {
            unsigned const m = (unsigned)(at & 15);
            if (m && (lane == 31 || next_key != key + 16)) b = __ldcs((uint4 const *)(src + (at & ~15ull) + 16));
            v = m ? grab_shift(a, b, m) : a;
            if (g.kind == kGrabBatch) v.x ^= p.flip, v.y ^= p.flip, v.z ^= p.flip, v.w ^= p.flip;
        } else if (!whole && d < p.total) {
            // the lane's bytes cross a segment end (or the end of the plan): byte by byte
            uint32_t w[4] = {0, 0, 0, 0};
            unsigned t = s;
#pragma unroll
            for (unsigned j = 0; j < 16; ++j) {
                unsigned long long const dj = d + j;
                if (dj >= p.total) continue;
                while (t + 1 < p.n_segs && p.segs[t + 1].dst <= dj) ++t;
                GrabSeg const &h = p.segs[t];
                unsigned byte = 0;
                if (h.kind == kGrabBatch) byte = (p.batch[h.src + (dj - h.dst)] ^ p.flip) & 0xffu;
                else if (h.kind == kGrabPrior) byte = p.prior[h.src + (dj - h.dst)];
                else if (h.kind == kGrabRing) byte = *(uint8_t const *)(h.src + (dj - h.dst));
                w[j >> 2] |= byte << (8 * (j & 3));
            }
            v.x = w[0], v.y = w[1], v.z = w[2], v.w = w[3];
        }
        __stcs(p.out + (d >> 4), v);
    }
}

// k_grab_ring: the last n bytes of a slot's chunk go to ring positions w0, w0 + 1, ... (mod the ring), as
// samp_grab_push() copies a block into its ring (src/samp_grab.c:63-88).  A lane stores one aligned 16-byte word of
// the ring: it loads the aligned source word, takes the one behind it from the next lane and shifts with
// __byte_perm, as k_grab does.  Only the words at the append's two ends go byte by byte; the ring's wrap needs no care,
// because aligned words never straddle it.  One pass: the bound is HBM, 2 x the bytes appended.
struct GrabRingSlot {
    unsigned long long src; // batch byte of the first appended byte
    unsigned n;             // bytes appended, <= kGrabRingBytes
    unsigned w0;            // their first ring position
};

struct GrabRingParams {
    uint8_t const *batch;   // 16-byte aligned
    uint8_t *rings;         // kGrabRingBytes per slot
    GrabRingSlot const *slots;
    unsigned ctas;          // per slot: the grid is n_slots x ctas
    unsigned flip;          // as GrabParams::flip
};

__global__ void __launch_bounds__(kGrabThreads) k_grab_ring(GrabRingParams p)
{
    unsigned const lane = threadIdx.x & 31;
    unsigned const s = blockIdx.x / p.ctas;
    unsigned long long const warp = ((unsigned long long)(blockIdx.x % p.ctas) * kGrabThreads + threadIdx.x) >> 5;
    unsigned long long const base = warp * (kGrabSpan / 16); // the warp's first word of the append
    {
        GrabRingSlot const q = p.slots[s];
        unsigned const m0 = q.w0 & 15;
        // from the word holding w0 on; a full ring from an unaligned w0 starts and ends in that one word
        unsigned long long const words = min((m0 + (unsigned long long)q.n + 15) / 16, (unsigned long long)kGrabRingBytes / 16);
        if (base >= words) return; // warp-uniform
        uint8_t *ring = p.rings + (unsigned long long)s * kGrabRingBytes;
        for (unsigned step = 0; step < kGrabSteps; ++step) {
            unsigned long long const w = base + step * 32u;
            if (w >= words) break; // warp-uniform
            unsigned long long const i = w + lane;
            long long const k = (long long)(i * 16) - (long long)m0; // append index of the word's first byte
            unsigned const ra = (unsigned)(((unsigned long long)(q.w0 - m0) + i * 16) % kGrabRingBytes);
            bool const live = i < words;
            bool const whole = live && k >= 0 && k + 16 <= (long long)q.n;
            unsigned long long const at = q.src + (unsigned long long)k;
            uint4 a = {0u, 0u, 0u, 0u};
            if (whole) a = __ldcs((uint4 const *)(p.batch + (at & ~15ull)));
            unsigned long long const key = whole ? (at & ~15ull) + 1 : 0ull;
            unsigned long long const next_key = __shfl_down_sync(0xffffffffu, key, 1);
            uint4 b;
            b.x = __shfl_down_sync(0xffffffffu, a.x, 1);
            b.y = __shfl_down_sync(0xffffffffu, a.y, 1);
            b.z = __shfl_down_sync(0xffffffffu, a.z, 1);
            b.w = __shfl_down_sync(0xffffffffu, a.w, 1);
            if (whole) {
                unsigned const m = (unsigned)(at & 15);
                if (m && (lane == 31 || next_key != key + 16)) b = __ldcs((uint4 const *)(p.batch + (at & ~15ull) + 16));
                uint4 v = m ? grab_shift(a, b, m) : a;
                v.x ^= p.flip, v.y ^= p.flip, v.z ^= p.flip, v.w ^= p.flip;
                __stcs((uint4 *)(ring + ra), v);
            } else if (live) {
                for (unsigned j = 0; j < 16; ++j) {
                    long long kk = k + j;
                    if (kk < 0) kk += kGrabRingBytes;
                    if (kk < (long long)q.n) ring[ra + j] = (uint8_t)(p.batch[q.src + (unsigned long long)kk] ^ p.flip);
                }
            }
        }
    }
}

} // namespace r433b
