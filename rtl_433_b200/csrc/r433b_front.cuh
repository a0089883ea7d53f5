// r433b_front.cuh -- k_front: IQ -> AM, one WARP per 2048-sample tile of a capture stream (sm_90a).
//
// The envelope low-pass y' = (a y + b (x + x')) >> 14 (src/baseband.c:145-169) is a floor map, not
// associative -- but it contracts by a / 2^14 = 0.854 per sample, so a trajectory started from ANY state is,
// after a few dozen samples of live signal, the true one.  Lane l of a warp owns the 64 consecutive samples
// [64 l, 64 l + 64) of its tile (one 128-byte line of cu8 IQ), starts kWarmAm samples in front of them from
// a guess (the local envelope), and runs ONE trajectory through warm-up and chunk.  The warp then VERIFIES:
// lane l's state at its chunk boundary must equal lane l-1's state at its chunk end; the lowest lane that
// fails (about one chunk in a thousand) redoes its chunk from its neighbour's end state, and so on.  After the
// loop the tile is consistent from lane 0's start state onward.  That state is exact for the first tile of a
// stream (reset_sdr_flow(): zero) and a guess for every other tile: k_detect, which walks the tiles of a
// stream in order, checks the first AM value of a tile against the last one of the tile before (the filter
// state IS its last output) and recomputes forward from there in the rare case they do not fit, until its
// values meet the stored ones again (r433b_detect.cuh).  So tiles are independent here: the grid is
// streams x tiles, every SM runs the same ~300 instructions, and the AM goes to HBM once (2 B per sample)
// together with the bounds of every 64-sample chunk.
//
// One envelope needs 2.5 instructions (xor + 2 and + 2 dp4a per pair of samples), one filter step 4.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/r433b.h"
#include "r433b_core.cuh"

#ifdef R433B_SIMT_EMU
#define R4_DYN_SMEM(type, name) type *name = reinterpret_cast<type *>(simt::st().dyn_smem)
#define R4_NOINLINE
// a chained chunk has no samples in front of its start: no stream index may go below 0
#define R4_EMU_ASSERT_POS(pos) assert((long long)(pos) >= 0)
#else
#define R4_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
#define R4_NOINLINE __noinline__
#define R4_EMU_ASSERT_POS(pos) ((void)0)
#endif

namespace r433b {

constexpr int kChunk = 64;                 // samples per lane per tile
constexpr int kTile = 32 * kChunk;         // 2048
#ifndef R4_WARM_AM
#define R4_WARM_AM 64
#endif
constexpr int kWarmAm = R4_WARM_AM;                // warm-up samples of the AM trajectory (multiple of 16, <= kChunk)
constexpr int kFrontWarps = 4;             // warps (tiles) per CTA of k_front
constexpr int kFrontCtasPerSm = 10;             // 48 registers; shared memory holds 11 (cu8) or 6 (cs16) CTAs per SM

// bounds of the AM values of one 64-sample chunk (they may be wider than the truth, never narrower)
struct ChunkInfo {
    int16_t cmin, cmax;
};

// Summary of one tile, enough for k_detect to rule a noise tile out without loading its AM (r433b_detect.cuh,
// idle_skip): bounds of the stored AM (wider than the truth or exact, never narrower), the stored AM of its first
// and last sample, and x[0] + x[-1] as the hand-over check feeds the filter (x[-1] narrowed at block starts).
struct alignas(16) TileInfo {
    int16_t tmin, tmax;
    int16_t first, last;
    int32_t xsum;
    int32_t pad;
};

// The exact FM filter state (y, xf) after sample pos - 1
struct FmState {
    unsigned long long pos;
    int y, xf;
};

// Everything one stream carries from one launch to the next: between the time slices of a batch, and between the
// chunks of a chained batch (r433b_process_chained), where a chunk ends on a block boundary and the next one starts
// its positions at 0 again (start_abs, fsk_offset and fm_state.pos are rebased by the chunk's length).
struct StreamState {
    DetState d;
    int y_am;
    FmState fm_state;
    unsigned log_n, last_start, last_count;
    unsigned seq;
    int flushed;      // the end of the stream's range (flush, or the end of a chunk of a file that goes on) is done
    FmState fm_start; // in front of the chunk: the FM filter state (pos 0) ...
    int iq_i, iq_q;   // ... and the last IQ sample of the previous chunk (centred); zero at a file start
};

// 16 contiguous bytes (8 cu8 / 4 cs16 samples) starting at sample `pos` of the stream: one 128-bit load;
// zero-filled past `n_valid` samples counted from pos.
template <int SS>
__device__ __forceinline__ void load_group(uint8_t const *src, unsigned long long pos, long long n_valid, unsigned flip,
        uint32_t (&rw)[4])
{
    constexpr int SPL = 16 / SS;
    R4_EMU_ASSERT_POS(pos);
    uint8_t const *g = src + pos * SS;
    if (n_valid >= SPL) {
        uint4 v = __ldg(reinterpret_cast<uint4 const *>(g));
        rw[0] = v.x ^ flip;
        rw[1] = v.y ^ flip;
        rw[2] = v.z ^ flip;
        rw[3] = v.w ^ flip;
    } else {
        rw[0] = rw[1] = rw[2] = rw[3] = 0u;
        int nb = n_valid > 0 ? (int)n_valid * SS : 0;
        for (int bidx = 0; bidx < nb; ++bidx) rw[bidx >> 2] |= (uint32_t)(g[bidx] ^ (flip & 0xff)) << (8 * (bidx & 3));
    }
}

// -Y magest on cu8 (src/baseband.c:65-79): rarely asked for, kept out of the hot loops' instruction stream
// (two magnitudes per returned word: they are below 2^15)
__device__ R4_NOINLINE uint4 mag_group_cu8(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3)
{
    auto two = [](uint32_t w) {
        return (uint32_t)mag_cu8((int)(w & 0xff), (int)((w >> 8) & 0xff))
                | ((uint32_t)mag_cu8((int)((w >> 16) & 0xff), (int)(w >> 24)) << 16);
    };
    uint4 r;
    r.x = two(w0);
    r.y = two(w1);
    r.z = two(w2);
    r.w = two(w3);
    return r;
}

// envelope / magnitude of the SPL samples of one group (src/baseband.c:36-45, :65-79, :96-110)
template <int SS>
__device__ __forceinline__ void env_group(uint32_t const (&rw)[4], int use_mag, int (&x)[16 / SS])
{
    if (SS == 2) {
        if (!use_mag) {
            // (127 - I)^2 + (127 - Q)^2: 127 - v is v ^ 0x7f read as a signed byte; one dp4a squares and adds a pair
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                uint32_t s = rw[w] ^ 0x7f7f7f7fu;
                x[2 * w] = __dp4a((int)s, (int)(s & 0x0000ffffu), 0);
                x[2 * w + 1] = __dp4a((int)s, (int)(s & 0xffff0000u), 0);
            }
        } else {
            uint4 const m = mag_group_cu8(rw[0], rw[1], rw[2], rw[3]);
            x[0] = (int)(m.x & 0xffff);
            x[1] = (int)(m.x >> 16);
            x[2] = (int)(m.y & 0xffff);
            x[3] = (int)(m.y >> 16);
            x[4] = (int)(m.z & 0xffff);
            x[5] = (int)(m.z >> 16);
            x[6] = (int)(m.w & 0xffff);
            x[7] = (int)(m.w >> 16);
        }
    } else {
#pragma unroll
        for (int j = 0; j < 16 / SS; ++j) {
            uint32_t w = rw[j & 3];
            x[j] = mag_cs16((int)(int16_t)(w & 0xffff), (int)(int16_t)(w >> 16));
        }
    }
}

// envelope / magnitude of ONE sample of the stream (cold paths: tile hand-over check and repair in k_detect)
template <int SS>
__device__ __forceinline__ int env_at(uint8_t const *src, unsigned long long pos, unsigned flip, int use_mag)
{
    R4_EMU_ASSERT_POS(pos);
    uint8_t const *g = src + pos * SS;
    if (SS == 2) {
        unsigned const w = (unsigned)*reinterpret_cast<uint16_t const *>(g) ^ (flip & 0xffff); // streams start 16-byte aligned
        int i = (int)(w & 0xff), q = (int)(w >> 8);
        return use_mag ? mag_cu8(i, q) : env_cu8(i, q);
    }
    uint32_t w = *reinterpret_cast<uint32_t const *>(g) ^ flip;
    return mag_cs16((int)(int16_t)(w & 0xffff), (int)(int16_t)(w >> 16));
}

// envelope / magnitude of a centred IQ sample (StreamState::iq_i / iq_q: the sample in front of a chained chunk)
template <int SS>
__device__ __forceinline__ int env_iq(int ci, int cq, int use_mag)
{
    if (SS == 2) return use_mag ? mag_cu8(ci + 128, cq + 128) : env_cu8(ci + 128, cq + 128);
    return mag_cs16(ci, cq);
}

// the centred IQ sample at `pos` (flip applied: cs8 reads as cu8)
template <int SS>
__device__ __forceinline__ void iq_at(uint8_t const *src, unsigned long long pos, unsigned flip, int &ci, int &cq)
{
    R4_EMU_ASSERT_POS(pos);
    uint8_t const *g = src + pos * SS;
    if (SS == 2) {
        ci = (int)(g[0] ^ (flip & 0xff)) - 128;
        cq = (int)(g[1] ^ (flip & 0xff)) - 128;
    } else {
        uint32_t w = *reinterpret_cast<uint32_t const *>(g) ^ flip;
        ci = (int)(int16_t)(w & 0xffff);
        cq = (int)(int16_t)(w >> 16);
    }
}

struct FrontParams {
    uint8_t const *data;
    unsigned long long const *offsets;    // bytes, n_streams + 1
    unsigned long long const *lengths;    // optional: bytes of stream i actually used
    unsigned long long const *am_offsets; // first sample of stream i in `am` (multiples of kTile), n_streams
    unsigned n_streams;
    unsigned long long tile_begin;        // the tiles [tile_begin, tile_begin + tiles) of every stream
    unsigned tiles;
    int use_mag;
    unsigned flip;                        // XOR mask applied to every loaded word: 0x80808080 turns cs8 into cu8
    unsigned block_samples;
    int a1, b0;
    int16_t *am;
    ChunkInfo *chunks;                    // one per 64 samples of `am`
    TileInfo *tile_info;                  // one per tile of `am`
    unsigned *counters;                   // [4] chunks done twice
    int spoil;                            // tests: 1 = lane 0's guess is made wrong, 2 = every lane's, 3 = lane 0's in every
                                          // 7th tile, 4 = lane 0's in every tile incl. tile 0 of a continued chunk
                                          // (R433B_SPOIL_FRONT)
    StreamState const *state;             // chained batches: the state carried in front of the chunk ...
    unsigned char const *cont;            // ... for the streams whose flag is set (nullptr: none)
};

// Shared-memory staging of one tile's IQ: the chunks [-kWarmChunks, 32) of the tile, every chunk (C samples)
// followed by 16 bytes of padding so that the lanes' 128-bit reads of their own chunks spread over all banks.
constexpr int kWarmChunks = (kWarmAm + kChunk - 1) / kChunk;
template <int SS>
struct FrontStage {
    static constexpr int kChunkBytes = kChunk * SS;
    static constexpr int kSlot = kChunkBytes + 16;
    static constexpr int kPieces = (32 + kWarmChunks) * (kChunkBytes / 16); // 16-byte pieces per tile
    static constexpr int kBytes = (32 + kWarmChunks) * kSlot;
    // byte offset in the stage of sample `rel` (relative to the tile start, >= -kWarmChunks * C), a multiple of 16 / SS
    static __device__ __forceinline__ int at(int rel) { return ((rel + kWarmChunks * kChunk) / kChunk) * kSlot + ((rel + kWarmChunks * kChunk) % kChunk) * SS; }
    // byte offset of the 16-bit AM of tile sample `rel` (>= 0): written over the IQ of the same chunk, behind the reads
    static __device__ __forceinline__ int out_at(int rel) { return (rel / kChunk + kWarmChunks) * kSlot + (rel % kChunk) * 2; }
};

// 16 bytes global -> shared, asynchronously; bytes past `valid` (0..16) are zero-filled
__device__ __forceinline__ void stage_piece(void *dst_smem, void const *src, int valid)
{
#ifdef R433B_SIMT_EMU
    uint8_t *d = reinterpret_cast<uint8_t *>(dst_smem);
    for (int i = 0; i < 16; ++i) d[i] = i < valid ? reinterpret_cast<uint8_t const *>(src)[i] : 0;
#else
    unsigned const d = (unsigned)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(valid) : "memory");
#endif
}
__device__ __forceinline__ void stage_wait()
{
#ifndef R433B_SIMT_EMU
    asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}

template <int SS>
__global__ void __launch_bounds__(kFrontWarps * 32, kFrontCtasPerSm) k_front(FrontParams p)
{
    constexpr int SPL = 16 / SS;
    constexpr int C = kChunk;
    using St = FrontStage<SS>;
    R4_DYN_SMEM(uint8_t, front_smem);
    int const lane = threadIdx.x & 31;
    unsigned long long const w = (unsigned long long)blockIdx.x * kFrontWarps + (threadIdx.x >> 5);
    unsigned const s = (unsigned)(w / p.tiles);
    if (s >= p.n_streams) return;
    unsigned long long const t0 = (p.tile_begin + w % p.tiles) * (unsigned long long)kTile;
    unsigned long long const byte0 = p.offsets[s];
    unsigned long long const N = (p.lengths ? p.lengths[s] : p.offsets[s + 1] - byte0) / SS;
    if (t0 >= N) return;
    uint8_t const *const src = p.data + byte0;
    unsigned long long const remain = N - t0;
    int const nv_tile = remain < (unsigned long long)kTile ? (int)remain : kTile;
    int const a1 = p.a1, b0 = p.b0;
    uint8_t *const stage = front_smem + (threadIdx.x >> 5) * St::kBytes;

    // ---- the tile's IQ (and the warm-up samples in front of it) into shared memory: coalesced 16-byte pieces,
    //      all of them in flight at once; nothing in front of the stream or past its end is touched ----
    {
        long long const first = (long long)t0 - kWarmChunks * C; // sample of piece 0
#pragma unroll 1
        for (int i = lane; i < St::kPieces; i += 32) {
            long long const smp = first + (long long)i * SPL;
            long long const left = (long long)N - smp; // samples of the stream from smp on
            int const valid = smp < 0 ? 0 : (left >= SPL ? 16 : (left > 0 ? (int)left * SS : 0));
            int const piece_in_chunk = i % (St::kChunkBytes / 16);
            int const chunk = i / (St::kChunkBytes / 16);
            stage_piece(stage + chunk * St::kSlot + piece_in_chunk * 16, valid ? src + smp * SS : src, valid);
        }
        stage_wait();
        __syncwarp();
    }
    auto group_at = [&](int rel, uint32_t (&rw)[4]) { // the SPL samples from tile sample `rel` on (a multiple of SPL)
        uint4 const v = *reinterpret_cast<uint4 const *>(stage + St::at(rel));
        rw[0] = v.x ^ p.flip;
        rw[1] = v.y ^ p.flip;
        rw[2] = v.z ^ p.flip;
        rw[3] = v.w ^ p.flip;
    };

    int const base = lane * C;
    int nv = nv_tile - base;
    nv = nv < 0 ? 0 : (nv > C ? C : nv);
    unsigned long long const gpos = t0 + (unsigned long long)base; // first sample of the chunk in the stream

    int y = 0, xp = 0;
    // the first sample of a continued chunk: the exact state the previous chunk ended with, as for a stream's first
    // tile (x[-1] is narrowed below: a chunk starts a block)
    bool const carried = gpos == 0 && p.cont && p.cont[s];
    if (carried) {
        y = p.state[s].y_am;
        xp = env_iq<SS>(p.state[s].iq_i, p.state[s].iq_q, p.use_mag);
    }
    if (gpos != 0 && nv > 0) { // reads the chunk in front of this lane's: before the __syncwarp() below
        uint32_t rw[4];
        int x[SPL];
        int g0 = -kWarmAm; // warm-up start relative to the chunk
        if (gpos >= (unsigned long long)kWarmAm) {
            // guess: the filter has (almost) unit gain, its state is near the local envelope
            group_at(base - kWarmAm, rw);
            env_group<SS>(rw, p.use_mag, x);
            xp = x[0];
            y = (x[0] + x[1]) >> 1;
            if (y > 32767) y = 32767;
        } else {
            g0 = -(int)gpos; // the warm-up begins at sample 0 of the stream: the reset state, exact
        }
#pragma unroll 2
        for (int g = g0; g < 0; g += SPL) {
            group_at(base + g, rw);
            env_group<SS>(rw, p.use_mag, x);
            // (a block start inside the warm-up is not modelled: the state is a guess anyway)
#pragma unroll
            for (int j = 0; j < SPL; ++j) {
                y = iir16_nowrap(y, a1, b0, x[j] + xp);
                xp = x[j];
            }
        }
    }
    // x[0] of the tile, for the tile summary
    int x0;
    {
        uint32_t rw[4];
        int x[SPL];
        group_at(0, rw);
        env_group<SS>(rw, p.use_mag, x);
        x0 = x[0];
    }
    // From here on a lane's AM overwrites its own chunk's IQ in the stage (no other lane reads that chunk again), and
    // the warp stores the whole tile at the end, whole lines per instruction.  Stored lane by lane (32 partial lines
    // 128 bytes apart per instruction), the tiles in flight overflow the 50 MB L2 of an H100.
    __syncwarp();
    // the reference keeps x[-1] as int16 across block calls (src/baseband.c:167): only the first sample of a
    // block sees the narrowed value, and block starts are tile starts
    if (gpos % p.block_samples == 0) xp = (int)(int16_t)xp;
    if (p.spoil && (gpos != 0 || (p.spoil == 4 && carried))
            && (p.spoil == 2 || (lane == 0 && (p.spoil == 1 || p.spoil == 4 || (p.spoil == 3 && t0 / kTile % 7 == 0)))))
        y = y > 16000 ? y - 999 : y + 999; // tests: force the redo / repair paths
    int const y_b = y, xp_b = xp;
    int y_end = y, cmin = 32767, cmax = 0;
    // verify / redo loop: a lane's state at its chunk boundary must be what its left neighbour ended with; the
    // lowest lane that fails runs its chunk again from that state.  cmin / cmax only ever widen: they stay bounds.
    int ys = y_b;
    bool run = true, fixed = false;
    for (;;) {
        if (run) {
            if (fixed) {
                // a chunk run again: its stage slot holds AM by now, so its IQ is staged again (L2 hits), every
                // piece in flight at once (cp.async does not block), zero-filled past the stream end like the first time
#pragma unroll 1
                for (int q = 0; q < St::kChunkBytes / 16; ++q) {
                    long long const smp = (long long)gpos + q * SPL;
                    long long const left = (long long)N - smp;
                    int const valid = left >= SPL ? 16 : (left > 0 ? (int)left * SS : 0);
                    stage_piece(stage + St::at(base + q * SPL), valid ? src + smp * SS : src, valid);
                }
                stage_wait();
            }
            int yy = ys, xx = xp_b;
            int k = 0;
#pragma unroll 2
            for (; k + SPL <= nv; k += SPL) {
                uint32_t rw[4];
                int x[SPL];
                uint32_t o[SPL / 2];
                group_at(base + k, rw);
                env_group<SS>(rw, p.use_mag, x);
#pragma unroll
                for (int j = 0; j < SPL; j += 2) {
                    int ya = iir16_nowrap(yy, a1, b0, x[j] + xx);
                    int yb = iir16_nowrap(ya, a1, b0, x[j + 1] + x[j]);
                    xx = x[j + 1];
                    yy = yb;
                    cmin = min(cmin, min(ya, yb));
                    cmax = max(cmax, max(ya, yb));
                    // AM dips below zero behind a full-scale sample at a block start (x[-1] narrowed to -32768):
                    // ya is cut to 16 bits so that its sign does not spill over yb
                    o[j >> 1] = (uint32_t)(uint16_t)ya | ((uint32_t)yb << 16);
                }
                if (SS == 2) {
                    uint4 v;
                    v.x = o[0];
                    v.y = o[1];
                    v.z = o[SPL / 2 > 2 ? 2 : 0];
                    v.w = o[SPL / 2 > 3 ? 3 : 0];
                    *reinterpret_cast<uint4 *>(stage + St::out_at(base + k)) = v;
                } else {
                    uint2 v;
                    v.x = o[0];
                    v.y = o[1];
                    *reinterpret_cast<uint2 *>(stage + St::out_at(base + k)) = v;
                }
            }
            if (k < nv) { // ragged end of the stream (the stage is zero-filled past it)
                uint32_t rw[4];
                int x[SPL];
                group_at(base + k, rw);
                env_group<SS>(rw, p.use_mag, x);
#pragma unroll
                for (int j = 0; j < SPL; ++j) {
                    if (k + j < nv) {
                        yy = iir16_nowrap(yy, a1, b0, x[j] + xx);
                        xx = x[j];
                        cmin = min(cmin, yy);
                        cmax = max(cmax, yy);
                        *reinterpret_cast<int16_t *>(stage + St::out_at(base + k + j)) = (int16_t)yy;
                    }
                }
            }
            y_end = yy;
        }
        int prev_end = __shfl_up_sync(0xffffffffu, y_end, 1);
        bool ok = lane == 0 || fixed || nv == 0 || y_b == prev_end;
        unsigned bad = __ballot_sync(0xffffffffu, !ok);
        if (!bad) break;
        int const f = __ffs(bad) - 1; // lanes below f are consistent with lane 0
        ys = __shfl_sync(0xffffffffu, y_end, f - 1);
        run = lane == f;
        if (run) {
            fixed = true;
            atomicAdd(&p.counters[4], 1u);
        }
    }
    __syncwarp();
    int16_t *const tile_out = p.am + p.am_offsets[s] + t0;
#pragma unroll 1
    for (int i = lane; i * 8 < nv_tile; i += 32) { // 16-byte pieces of 8 AM values
        int const smp = i * 8;
        uint8_t const *const sp = stage + St::out_at(smp);
        if (smp + 8 <= nv_tile)
            *reinterpret_cast<uint4 *>(tile_out + smp) = *reinterpret_cast<uint4 const *>(sp);
        else
            for (int j = 0; j < nv_tile - smp; ++j) tile_out[smp + j] = reinterpret_cast<int16_t const *>(sp)[j];
    }
    ChunkInfo ci;
    ci.cmin = (int16_t)(nv > 0 ? cmin : 32767);
    ci.cmax = (int16_t)(nv > 0 ? cmax : 0);
    p.chunks[(p.am_offsets[s] + gpos) / C] = ci;
    int const tmin = __reduce_min_sync(0xffffffffu, nv > 0 ? cmin : 32767);
    int const tmax = __reduce_max_sync(0xffffffffu, nv > 0 ? cmax : -32768);
    int const last = __shfl_sync(0xffffffffu, y_end, (nv_tile - 1) / C);
    if (lane == 0) {
        TileInfo ti;
        ti.tmin = (int16_t)tmin;
        ti.tmax = (int16_t)tmax;
        ti.first = *reinterpret_cast<int16_t const *>(stage + St::out_at(0));
        ti.last = (int16_t)last;
        ti.xsum = x0 + xp_b; // lane 0's x[-1]: narrowed above when the tile starts a block
        ti.pad = 0;
        p.tile_info[(p.am_offsets[s] + t0) / kTile] = ti;
    }
}

} // namespace r433b
