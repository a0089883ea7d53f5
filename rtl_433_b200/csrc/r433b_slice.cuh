// r433b_slice.cuh -- the pulse slicers (pulse train -> bitbuffer rows) and the compact event
// encoder they write through.  __host__ __device__ inlines: device code in r433b_kernels.cu,
// CPU-side unit tests through tests/host_core.cpp.
//
// One slicer run = one (package, device) pair, executed by one thread; the 32 lanes of a warp
// are 32 devices looking at the SAME package.  To keep those lanes converged every slicer is
// split into a small per-modulation "front end" that turns one pulse (or symbol) into a fixed
// record of bit-buffer operations (Step: runs of ones/zeros, a row operation, a single bit, an
// emit condition, trailing zeros -- always in that order) and ONE shared "back end" that applies
// the record to the event writer.  Lanes of different devices then differ only in predicates.
//
// Instead of building a 6604-byte bitbuffer_t (include/bitbuffer.h:34-40) per event, rows are
// streamed straight into the pair's private output region in the wire format below; the host
// re-inflates a real bitbuffer_t only when it calls a decoder (r433b_host.hpp).  Every run is
// executed twice by the kernel: once counting (size), once storing.
//
//   event   := u32 { num_rows:7, dirty:1, free_row:8, words:16 }   words = whole event incl. this
//              row*  [u32 last_row_words  -- only if dirty]
//   row     := u32 { bits:16, syncs:16 }  then ceil(bits/32) data words (physical row order;
//              bit i of the row is bit (7 - i%8) of byte i/8, exactly bitbuffer_t's bb layout)
//
// `dirty` marks the reference's 50-row overflow path, which zeroes the last row's length but
// keeps its bytes (src/bitbuffer.c:118-121): the number of data words then comes from the trailer.
#pragma once
#include <stdint.h>
#include "r433b_core.cuh"

namespace r433b {

constexpr int kBbRows = 50;   // include/bitbuffer.h:28
constexpr int kBbCols = 128;  // include/bitbuffer.h:27

// float helpers: no fused multiply-add anywhere (the reference is built without contraction)
#ifdef __CUDA_ARCH__
R4_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
R4_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
R4_HD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
R4_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
R4_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
#else
R4_HD float fmul(float a, float b) { volatile float r = a * b; return r; }
R4_HD float fadd(float a, float b) { volatile float r = a + b; return r; }
R4_HD float fdiv(float a, float b) { volatile float r = a / b; return r; }
R4_HD double dadd(double a, double b) { volatile double r = a + b; return r; }
R4_HD double dmul(double a, double b) { volatile double r = a * b; return r; }
#endif

// Integer timing of one device at one sample rate.  Derived ON THE HOST (r433b_host.cpp) with
// the reference's float expressions (src/pulse_slicer.c:70-91) and shipped as integers.
struct SlicerParams {
    int modulation;
    int ok; // bit 0: all six scaled widths survived (the check of every slicer but RZI, src/pulse_slicer.c:79-84);
            // bit 1: short/long/reset survived (RZI's check, :877-879).  A clear bit = "sample rate too low": no events
    int s_short, s_long, s_reset, s_gap, s_sync, s_tol;
    float f_short, f_long; // 1/(width*samples_per_us) or 0
    unsigned priority;
    int gate; // decoder length gate (r433b_gate.min_bits): events with >= 1 row whose rows all hold fewer bits are
              // counted, not stored; 0 = every event is stored
};

// ----------------------------------------------------------------------------- writer ----

R4_HD uint32_t bswap32(uint32_t v)
{
#ifdef __CUDA_ARCH__
    return __byte_perm(v, 0, 0x0123);
#else
    return (v >> 24) | ((v >> 8) & 0xff00u) | ((v << 8) & 0xff0000u) | (v << 24);
#endif
}

// One writer type serves both passes: out == nullptr only counts.  All offsets are in 32-bit
// words; every store is one aligned word.  Bits are gathered MSB-first in `acc` (bit i of the
// row at position 31 - i%32) and byte-swapped on store, which yields bitbuffer_t's layout
// (bit i in byte i/8 at position 7 - i%8) in little-endian memory.
struct EventWriter {
    uint32_t *out;      // pair region, or nullptr while counting
    unsigned limit;     // words the counting pass committed: rows of a trailing, never-emitted
                        // event lie beyond it and must not be written

    unsigned pos;       // words used by finished events + the current event so far
    unsigned committed; // words up to the end of the last emitted event
    unsigned events;
    // current event
    unsigned ev_start;
    unsigned num_rows, free_row;
    unsigned row0_bits; // bits_per_row[0] once row 0 is closed
    // current (last) row
    unsigned row_hdr;   // word offset of its header
    unsigned bits, syncs;
    unsigned row_hw;    // data words that hold something
    uint32_t acc;       // word being assembled (MSB first)
    bool dirty;         // row length was reset while its bytes stayed (50-row overflow path)
    // decoder length gate (SURVEY 8(f1)): an event the decoder would turn down for its row lengths alone is
    // counted instead of stored -- by row count, because many decoders look at num_rows first
    unsigned gate;      // bits; 0 = off
    unsigned max_bits;  // longest closed row of the current event
    unsigned gated1, gatedN; // dropped events of one row / of several rows

    R4_HD void init(uint32_t *o, unsigned region_words = 0, unsigned gate_bits = 0)
    {
        out = o;
        limit = region_words;
        pos = committed = 0;
        events = 0;
        gate = gate_bits;
        gated1 = gatedN = 0;
        reset_event();
    }

    R4_HD void reset_event() // bitbuffer_clear(), src/bitbuffer.c:17
    {
        pos = committed;
        ev_start = committed;
        num_rows = free_row = 0;
        row0_bits = 0;
        row_hdr = 0;
        bits = syncs = row_hw = 0;
        acc = 0;
        dirty = false;
        max_bits = 0;
    }

    R4_HD void put(unsigned at, uint32_t v)
    {
        if (out && at < limit) out[at] = v;
    }

    R4_HD unsigned first_row_bits() const { return num_rows <= 1 ? bits : row0_bits; }
    R4_HD unsigned last_row_bits() const { return bits; }

    R4_HD void open_row()
    {
        row_hdr = pos;
        pos += 1;
        bits = syncs = row_hw = 0;
        acc = 0;
    }

    R4_HD void flush_word()
    {
        unsigned w = (bits - 1) >> 5; // the word holding the newest bit
        unsigned at = row_hdr + 1 + w;
        if (out && at < limit) {
            uint32_t v = bswap32(acc);
            if (w < row_hw)
                out[at] |= v;
            else
                out[at] = v;
        }
        if (w + 1 > row_hw) row_hw = w + 1;
        acc = 0;
    }

    R4_HD void close_row()
    {
        if (bits & 31) flush_word();
        put(row_hdr, bits | (syncs << 16));
        pos = row_hdr + 1 + row_hw;
    }

    R4_HD void first_row() // "Add first row automatically", src/bitbuffer.c:24-26
    {
        if (num_rows == 0) {
            ev_start = pos;
            pos += 1;
            num_rows = free_row = 1;
            open_row();
        }
    }

    // `count` calls of bitbuffer_add_bit(bits, value), src/bitbuffer.c:22-56, a word at a time
    R4_HD void add_bits(int value, int count)
    {
        first_row();
        {
            // common case: the run ends inside the current word and the row neither starts on nor
            // crosses a 1024-bit spill boundary, nor comes near the 65535-bit limit
            unsigned const p = bits & 31, in_row = bits & (kBbCols * 8 - 1);
            if ((unsigned)count <= 32 - p && (in_row != 0 || bits == 0) && bits < 60000u) {
                if (value) acc |= (0xffffffffu >> (32 - count)) << (32 - p - count);
                bits += (unsigned)count;
                if ((bits & 31) == 0) flush_word();
                return;
            }
        }
        while (count > 0) {
            if (bits == 65535u) return; // row length limit: further bits are dropped
            if (bits > 0 && (bits & (kBbCols * 8 - 1)) == 0) { // spill into the next physical row
                if (free_row < (unsigned)kBbRows)
                    free_row++;
                else
                    return; // no room: this and all following bits of the run are dropped
            }
            unsigned p = bits & 31;
            unsigned room = 32 - p; // never crosses a 1024-bit boundary either
            unsigned n = (unsigned)count < room ? (unsigned)count : room;
            if (bits + n > 65535u) n = 65535u - bits;
            if (value) acc |= (n == 32 ? 0xffffffffu : ((1u << n) - 1u)) << (room - n);
            bits += n;
            count -= (int)n;
            if ((bits & 31) == 0) flush_word();
        }
    }

    R4_HD void add_bit(int bit) { add_bits(bit, 1); }

    // src/bitbuffer.c:106-122
    R4_HD void add_row()
    {
        first_row();
        if (free_row < (unsigned)kBbRows) {
            if (num_rows == 1) row0_bits = bits;
            if (bits > max_bits) max_bits = bits;
            close_row();
            free_row++;
            // physical rows taken by spill-over sit between the old and the new last row
            for (unsigned r = num_rows; r + 1 < free_row; ++r) {
                put(pos, 0);
                pos += 1;
            }
            num_rows = free_row;
            open_row();
        } else {
            // row count exhausted: length forgotten, bytes (and syncs) stay
            if (bits & 31) flush_word();
            bits = 0;
            dirty = true;
            acc = 0;
        }
    }

    // src/bitbuffer.c:124-133
    R4_HD void add_sync()
    {
        first_row();
        if (bits) add_row();
        syncs++;
    }

    // account_event(): hand the buffer to the decoder, then clear it (src/pulse_slicer.c:26-66)
    R4_HD void emit()
    {
        if (num_rows == 0) { // an empty buffer is still an event (e.g. nrzs): header only
            ev_start = pos;
            pos += 1;
        } else if ((bits > max_bits ? bits : max_bits) < gate) {
            // bits_per_row[] all below the decoder's gate: decode_fn would return the gate's code at once
            if (num_rows == 1) gated1++; else gatedN++;
            reset_event();
            return;
        } else {
            close_row();
            if (dirty) { // only the last row can be: its data length travels in a trailer word
                put(pos, row_hw);
                pos += 1;
            }
        }
        put(ev_start, num_rows | (dirty ? 0x80u : 0u) | (free_row << 8) | ((pos - ev_start) << 16));
        committed = pos;
        events++;
        reset_event();
    }
};

// ---------------------------------------------------------------------------- slicers ----

struct PulseView {
    int const *pulse;
    int const *gap;
    unsigned n;
};

enum { // include/r_device.h:24-40
    kModOokMc = 3, kModOokPcm = 4, kModOokPpm = 5, kModOokPwm = 6, kModOokPiwmRaw = 8, kModOokDmc = 9,
    kModOokOsv1 = 10, kModOokPiwmDc = 11, kModOokNrzs = 12, kModOokRzi = 13,
    kModFskPcm = 16, kModFskPwm = 17, kModFskMc = 18
};

// does run_ook_demods / run_fsk_demods (src/r_api.c:438-550) hand this package type to this device?
R4_HD bool device_takes(int modulation, int package_type)
{
    if (package_type == 1) return modulation >= 3 && modulation <= 13 && modulation != 7;
    return modulation >= 16 && modulation <= 18;
}

R4_HD int iabs(int v) { return v < 0 ? -v : v; }
R4_HD bool within(int v, int nominal, int tol) { return v >= nominal - tol && v <= nominal + tol; }
R4_HD int symbol_at(PulseView const &p, unsigned k) { return (k & 1) ? p.gap[k >> 1] : p.pulse[k >> 1]; } // src/pulse_slicer.c:529-535

// What one iteration of a slicer's main loop does to the bit buffer, in this fixed order.
enum { kRowNone = 0, kRowAdd, kRowSync, kRowClear, kRowIfOpen };
enum { kEmitNone = 0, kEmitAlways, kEmitIfRows, kEmitIfData, kEmitIfRow0, kEmitElseRowIfOpen };
struct Step {
    int ones;       // 1. run of one-bits
    int zeros;      // 2. run of zero-bits
    int row;        // 3. kRow*: add_row / add_sync / clear / add_row if the last row has bits
    int bit;        // 4. single bit: 0 none, 1 -> add_bit(0), 2 -> add_bit(1)
    int emit;       // 5. kEmit*: condition under which the event is handed over
    bool stop_if_emitted, clear_after;
    int post_zeros; // 6. zero-bits after a (non-stopping) emit decision
};

// Per-run state of the front ends (a union in spirit: each slicer uses a few fields)
struct SlicerState {
    unsigned k, total;     // loop index / bound (pulses, or symbols for the PIWM/DMC family)
    int b0, b1, b2, b3, b4, b5; // PWM / PPM class bounds
    float f_short, f_long; // PCM tuned reciprocals
    int i0, i1, i2;        // gap_limit / max_zeros / tol (PCM); lo / hi (MC); half_hi (OSV1); s_base (RZI)
    int since;             // MC: time since last edge; OSV1: manchester phase; RZI: fresh flag
    double edge;           // MC: 1.5 * s_short
    bool pending;          // OSV1: a zero bit owed before the first data pulse
    int cv, cg;            // pulse[k], gap[k] of the per-pulse slicers, loaded one step ahead (slicer_advance)
};

// Move a per-pulse slicer to pulse `k` and issue the loads of its widths now: they are needed one whole step (the
// front end's classification and the bit writer's work) later, so their latency -- every lane reads another package in
// k_slice2 -- is off the critical path.
R4_HD void slicer_advance(PulseView const &p, SlicerState &st, unsigned k)
{
    st.k = k;
    if (k < st.total) {
        st.cv = p.pulse[k];
        st.cg = p.gap[k];
    }
}

// ---- set-up: everything the reference does before its main loop; returns false if the slicer
//      produces nothing (src/pulse_slicer.c, "check for rounding to zero" and early returns)
// MOD: the modulation as a compile-time constant (kModAny = look at t.modulation).  A warp of k_slice2 runs one device,
// so slice_dispatch() picks the loop specialised for its slicer: the other front ends, and every Step field that slicer
// never sets, fold away in slicer_apply().
constexpr int kModAny = -1;
template <int MOD>
R4_HD int slicer_family(SlicerParams const &t)
{
    if (MOD != kModAny) return MOD;
    int const m = t.modulation; // the FSK variants share the front ends of their OOK counterparts
    return m == kModFskPwm ? (int)kModOokPwm : m == kModFskPcm ? (int)kModOokPcm : m == kModFskMc ? (int)kModOokMc : m;
}

template <int MOD>
R4_HD bool slicer_begin0(PulseView const &p, SlicerParams const &t, SlicerState &st)
{
    st.k = 0;
    st.cv = st.cg = 0;
    st.total = p.n;
    st.since = 0;
    st.pending = false;
    int const big = 0x7fffffff;
    switch (slicer_family<MOD>(t)) {
    case kModOokPwm: { // src/pulse_slicer.c:369-413; b0..b5 = one/zero/sync lo,hi
        if (!(t.ok & 1)) return false;
        st.b4 = st.b5 = 0;
        if (t.s_tol > 0) {
            st.b0 = t.s_short - t.s_tol; st.b1 = t.s_short + t.s_tol;
            st.b2 = t.s_long - t.s_tol;  st.b3 = t.s_long + t.s_tol;
            if (t.s_sync > 0) { st.b4 = t.s_sync - t.s_tol; st.b5 = t.s_sync + t.s_tol; }
        } else if (t.s_sync <= 0) {
            st.b0 = 0; st.b1 = (t.s_short + t.s_long) / 2 + 1;
            st.b2 = st.b1 - 1; st.b3 = big;
        } else if (t.s_sync < t.s_short) {
            st.b4 = 0; st.b5 = (t.s_sync + t.s_short) / 2 + 1;
            st.b0 = st.b5 - 1; st.b1 = (t.s_short + t.s_long) / 2 + 1;
            st.b2 = st.b1 - 1; st.b3 = big;
        } else if (t.s_sync < t.s_long) {
            st.b0 = 0; st.b1 = (t.s_short + t.s_sync) / 2 + 1;
            st.b4 = st.b1 - 1; st.b5 = (t.s_sync + t.s_long) / 2 + 1;
            st.b2 = st.b5 - 1; st.b3 = big;
        } else {
            st.b0 = 0; st.b1 = (t.s_short + t.s_long) / 2 + 1;
            st.b2 = st.b1 - 1; st.b3 = (t.s_long + t.s_sync) / 2 + 1;
            st.b4 = st.b3 - 1; st.b5 = big;
        }
        return true;
    }
    case kModOokPpm: { // :291-308; b0..b5 = zero/one/sync lo,hi
        if (!(t.ok & 1)) return false;
        st.b4 = st.b5 = 0;
        if (t.s_tol > 0) {
            st.b0 = t.s_short - t.s_tol; st.b1 = t.s_short + t.s_tol;
            st.b2 = t.s_long - t.s_tol;  st.b3 = t.s_long + t.s_tol;
            if (t.s_sync > 0) { st.b4 = t.s_sync - t.s_tol; st.b5 = t.s_sync + t.s_tol; }
        } else {
            st.b0 = 0;
            st.b1 = (t.s_short + t.s_long) / 2 + 1;
            st.b2 = st.b1 - 1;
            st.b3 = t.s_gap ? t.s_gap : t.s_reset;
        }
        return true;
    }
    case kModOokPcm: { // :89-214, the bit-period estimators
        if (!(t.ok & 1) || t.s_long == 0) return false;
        float f_short = t.f_short, f_long = t.f_long;
        int const gap_limit = t.s_gap ? t.s_gap : t.s_reset;
        int tol = t.s_tol;
        if (tol <= 0) tol = t.s_long / 4;
        bool const rz = t.s_short != t.s_long;
        int need = rz ? 4 : 12;
        int preamble = 0;
        unsigned const N = p.n;
        if (rz) {
            for (unsigned n = 0; n < N; ++n) { // :105-132
                int sw = 0, lw = 0, cnt = 0;
                while (n < N && within(p.pulse[n], t.s_short, tol) && within(p.pulse[n] + p.gap[n], t.s_long, tol)) {
                    sw += p.pulse[n];
                    lw += p.pulse[n] + p.gap[n];
                    cnt++;
                    n++;
                }
                if (cnt >= need) {
                    f_long = fdiv((float)cnt, (float)lw);
                    f_short = fdiv((float)cnt, (float)sw);
                    need = cnt;
                    preamble = cnt;
                }
            }
            if (preamble == 0) { // :134-157
                int sw = 0, lw = 0, cnt = 0;
                for (unsigned n = 0; n < N; ++n) {
                    if (within(p.pulse[n], t.s_short, tol) && within(p.pulse[n] + p.gap[n], t.s_long, tol)) {
                        sw += p.pulse[n];
                        lw += p.pulse[n] + p.gap[n];
                        cnt++;
                    }
                }
                if (cnt > 8) {
                    f_long = fdiv((float)cnt, (float)lw);
                    f_short = fdiv((float)cnt, (float)sw);
                }
            }
        } else {
            for (unsigned n = 0; n < N; ++n) { // :159-180, float product then DOUBLE +0.5
                int wsum = 0, cnt = 0;
                while (n < N && (int)dadd((double)fmul((float)p.pulse[n], f_short), 0.5) == 1
                        && (int)dadd((double)fmul((float)p.gap[n], f_long), 0.5) == 1) {
                    wsum += p.pulse[n] + p.gap[n];
                    cnt += 2;
                    n++;
                }
                if (cnt >= need) {
                    f_short = f_long = fdiv((float)cnt, (float)wsum);
                    need = cnt;
                    preamble = cnt;
                }
            }
            if (preamble == 0) { // :182-214
                int wsum = 0, cnt = 0;
                for (unsigned n = 0; n < N; ++n) {
                    if (within(p.pulse[n], t.s_short, tol)) { wsum += p.pulse[n]; cnt += 1; }
                    if (within(p.pulse[n], 2 * t.s_short, tol)) { wsum += p.pulse[n]; cnt += 2; }
                    if (within(p.gap[n], t.s_long, tol)) { wsum += p.gap[n]; cnt += 1; }
                    if (within(p.gap[n], 2 * t.s_long, tol)) { wsum += p.gap[n]; cnt += 2; }
                }
                if (cnt > 20) f_short = f_long = fdiv((float)cnt, (float)wsum);
            }
        }
        st.f_short = f_short;
        st.f_long = f_long;
        st.i0 = gap_limit;
        st.i1 = gap_limit / t.s_long; // max_zeros
        st.i2 = tol;
        return true;
    }
    case kModOokMc: // :451-478
        if (!(t.ok & 1)) return false;
        st.edge = dmul((double)t.s_short, 1.5);
        st.i0 = t.s_short - t.s_tol;
        st.i1 = t.s_short * 2 + t.s_tol;
        st.pending = true; // "First rising edge is always counted as a zero"
        return true;
    case kModOokDmc: case kModOokPiwmRaw: case kModOokPiwmDc:
        if (!(t.ok & 1)) return false;
        st.total = p.n * 2;
        return true;
    case kModOokNrzs:
        return (t.ok & 1) && t.s_short != 0;
    case kModOokOsv1: { // :797-835: twelve preamble pulses, a sync, then manchester data
        if (!(t.ok & 1)) return false;
        int const half_lo = t.s_short / 2, half_hi = t.s_short * 3 / 2, sync_lo = 2 * half_hi;
        int pre = 0;
        unsigned n;
        for (n = 0; n < p.n; ++n) {
            if (p.pulse[n] > half_lo && p.gap[n] > half_lo) {
                pre++;
                if (p.gap[n] > half_hi) break;
            } else {
                return false;
            }
        }
        if (pre != 12) return false;
        ++n;
        if (n >= (unsigned)kMaxPulses) return false; // the reference reads past the array here
        // n may equal num_pulses: the entry after the last pulse is part of the package record
        if (p.pulse[n] < sync_lo || p.gap[n] < sync_lo) return false;
        st.since = 0; // manchester phase
        if (p.gap[n] > p.pulse[n]) {
            st.since = 1;
            st.pending = true;
        }
        st.k = n + 1;
        st.i0 = half_hi;
        return true;
    }
    case kModOokRzi: // :866-885 (its rate check only looks at short/long/reset: `ok` bit 1)
        if (!(t.ok & 2) || t.s_long == 0) return false;
        st.i0 = t.s_long - t.s_short;
        st.since = 1; // at_start
        return true;
    default:
        return false;
    }
}

template <int MOD>
R4_HD bool slicer_begin(PulseView const &p, SlicerParams const &t, SlicerState &st)
{
    if (!slicer_begin0<MOD>(p, t, st)) return false;
    slicer_advance(p, st, st.k); // widths of the first pulse the main loop looks at
    return true;
}

// ---- one iteration of the main loop of the slicer -> what it does to the bit buffer
template <int MOD>
R4_HD Step slicer_step(PulseView const &p, SlicerParams const &t, SlicerState &st)
{
    Step s;
    s.ones = s.zeros = s.post_zeros = 0;
    s.row = kRowNone;
    s.bit = 0;
    s.emit = kEmitNone;
    s.stop_if_emitted = s.clear_after = false;
    unsigned const n = st.k;
    switch (slicer_family<MOD>(t)) {
    case kModOokPwm: { // src/pulse_slicer.c:415-447
        int v = st.cv, g = st.cg;
        if (v > st.b0 && v < st.b1) s.ones = 1;
        else if (v > st.b2 && v < st.b3) s.zeros = 1;
        else if (v > st.b4 && v < st.b5) s.row = kRowSync;
        else if (v <= st.b0) { }
        else s.row = kRowAdd;
        if (n == st.total - 1 || g > t.s_reset) s.emit = kEmitIfRows;
        else if (t.s_gap > 0 && g > t.s_gap) s.emit = kEmitElseRowIfOpen;
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokPpm: { // :310-335
        int g = st.cg;
        if (g > st.b0 && g < st.b1) s.zeros = 1;
        else if (g > st.b2 && g < st.b3) s.ones = 1;
        else if (g > st.b4 && g < st.b5) s.row = kRowSync;
        else if (g < t.s_reset) s.row = kRowAdd;
        if (n == st.total - 1 || g >= t.s_reset) s.emit = kEmitIfData;
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokPcm: { // :216-257
        int v = st.cv, g = st.cg;
        int highs = (int)fadd(fmul((float)v, st.f_short), 0.5f);
        int lows = (int)fadd(fmul((float)(g + t.s_short - t.s_long), st.f_long), 0.5f);
        if (lows > st.i1) lows = st.i1;
        s.ones = highs > 0 ? highs : 0;
        s.zeros = lows > 0 ? lows : 0;
        if (t.s_short != t.s_long && iabs(v - t.s_short) > st.i2) s.row = kRowClear;
        else if (g > st.i0 && g <= t.s_reset) s.row = kRowAdd;
        if (n == st.total - 1 || g > t.s_reset) s.emit = kEmitIfData;
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokMc: { // :478-525; the buffer always holds >= 1 row here
        if (st.pending) { // bitbuffer_add_bit(&bits, 0) in front of the loop
            st.pending = false;
            s.zeros = 1;
            break;
        }
        int v = st.cv, g = st.cg;
        int const lo = st.i0, hi = st.i1;
        if (t.s_tol > 0 && (v < lo || v > hi || g < lo || g > hi)) {
            if ((double)v > st.edge && v <= hi) s.ones = 1;
            s.row = kRowAdd;
            s.bit = 1;
            st.since = 0;
        } else if ((double)(v + st.since) > st.edge) {
            s.ones = 1;
            st.since = 0;
        } else {
            st.since += v;
        }
        if (n == st.total - 1 || g > t.s_reset) {
            s.emit = kEmitIfRows;
            s.post_zeros = 1;
            st.since = 0;
        } else if ((double)(g + st.since) > st.edge) {
            s.post_zeros = 1;
            st.since = 0;
        } else {
            st.since += g;
        }
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokDmc: { // :562-592 (consumes a second symbol after a short one)
        unsigned k = n;
        int sym = symbol_at(p, k);
        if (iabs(sym - t.s_short) < t.s_tol) {
            s.ones = 1;
            sym = k + 1 < st.total ? symbol_at(p, ++k) : 0;
            if (iabs(sym - t.s_short) > t.s_tol) {
                if (sym >= t.s_reset - t.s_tol)
                    k--;
                else
                    s.row = kRowIfOpen;
            }
        } else if (iabs(sym - t.s_long) < t.s_tol) {
            s.zeros = 1;
        } else if (sym >= t.s_reset - t.s_tol) {
            s.emit = kEmitIfRows;
        }
        st.k = k + 1;
        break;
    }
    case kModOokPiwmRaw: { // :627-654
        int sym = symbol_at(p, n);
        int cnt = (int)dadd((double)fmul((float)sym, t.f_short), 0.5);
        if (sym > t.s_long) {
            s.row = kRowAdd;
        } else if (iabs(sym - cnt * t.s_short) < t.s_tol) {
            if (cnt > 0) {
                if (n & 1) s.zeros = cnt; else s.ones = cnt;
            }
        } else if (sym < t.s_reset) {
            s.row = kRowIfOpen;
        }
        if (n == st.total - 1 || sym > t.s_reset) s.emit = kEmitIfRows;
        st.k = n + 1;
        break;
    }
    case kModOokPiwmDc: { // :684-710
        int sym = symbol_at(p, n);
        if (iabs(sym - t.s_short) < t.s_tol) s.ones = 1;
        else if (iabs(sym - t.s_long) < t.s_tol) s.zeros = 1;
        else if (sym < t.s_reset) s.row = kRowIfOpen;
        if (n == st.total - 1 || sym > t.s_reset) s.emit = kEmitIfRows;
        st.k = n + 1;
        break;
    }
    case kModOokNrzs: { // :741-756
        int v = st.cv;
        if (v > t.s_short) {
            s.ones = v / t.s_short;
            s.zeros = 1;
        } else if (v < t.s_short) {
            s.zeros = 1;
        }
        if (n == st.total - 1 || st.cg >= t.s_reset) s.emit = kEmitAlways;
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokOsv1: { // :837-862
        if (st.pending) { // a data bit hidden in the sync gap
            st.pending = false;
            s.zeros = 1;
            break;
        }
        int man = st.since;
        man ^= 1;
        if (man) s.ones++;
        if (st.cv > st.i0) {
            man ^= 1;
            if (man) s.ones++;
        }
        if (n == st.total - 1 || st.cg > t.s_reset) {
            s.emit = kEmitIfRows;
            s.stop_if_emitted = true;
        }
        man ^= 1;
        if (man) s.post_zeros++;
        if (st.cg > st.i0) {
            man ^= 1;
            if (man) s.post_zeros++;
        }
        st.since = man;
        slicer_advance(p, st, n + 1);
        break;
    }
    case kModOokRzi: { // :887-915
        int high = st.cv;
        int ones = st.since ? (high + t.s_long / 2) / t.s_long : (high - st.i0 + t.s_long / 2) / t.s_long;
        st.since = 0;
        s.ones = ones > 0 ? ones : 0;
        if (st.cg > t.s_reset || n == st.total - 1) {
            s.emit = kEmitIfRow0;
            s.clear_after = true;
            st.since = 1;
        } else {
            s.post_zeros = 1;
        }
        slicer_advance(p, st, n + 1);
        break;
    }
    default:
        st.k = st.total;
        break;
    }
    return s;
}

// ---- the shared back end.  Returns false when the slicer is finished (OSV1 after its event).
// The 32 lanes of a warp are 32 devices that want different things from the writer at the same pulse; whatever
// any lane wants is executed by the warp, so every writer primitive has ONE call site here and the lanes'
// differences are predicates in front of it: a one bit and a zero bit are the same add_bits() with another value,
// add_row / add_sync / "row if open" / "else row if open" are one add_row() with another condition.
template <class W>
R4_HD bool slicer_apply(Step const &s, W &w)
{
    // 1./2. the runs of bits: most slicers produce ones OR zeros per step (PCM and NRZS both, ones first)
    {
        int const first = s.ones ? s.ones : s.zeros;
        if (first) w.add_bits(s.ones ? 1 : 0, first);
        if (s.ones && s.zeros) w.add_bits(0, s.zeros);
    }
    // 3. the row operation, and the one a step with kEmitElseRowIfOpen would do in 5.: never both (a row just
    //    added is empty, which is what "if open" tests), and the steps that carry one of them have no `bit` in
    //    between, so the second condition can be evaluated here
    if (s.row == kRowAdd || s.row == kRowSync) w.first_row();
    bool const open = w.num_rows > 0 && w.last_row_bits() > 0;
    bool const want_row = s.row == kRowAdd || (s.row == kRowSync && w.last_row_bits() > 0)
            || ((s.row == kRowIfOpen || s.emit == kEmitElseRowIfOpen) && open);
    if (want_row) w.add_row();
    if (s.row == kRowSync) w.syncs++; // bitbuffer_add_sync(): new row if the last one has bits, then count
    if (s.row == kRowClear) w.reset_event();
    // 4. single bit (Manchester's invalid-width path)
    if (s.bit) w.add_bits(s.bit - 1, 1);
    // 5. hand the event over?
    bool go = false;
    if (s.emit == kEmitAlways) go = true;
    else if (s.emit == kEmitIfRows) go = w.num_rows > 0;
    else if (s.emit == kEmitIfData) go = w.first_row_bits() > 0 || w.num_rows > 1;
    else if (s.emit == kEmitIfRow0) go = w.first_row_bits() > 0;
    if (go) w.emit();
    if (s.clear_after) w.reset_event();
    if (go && s.stop_if_emitted) return false;
    // 6.
    if (s.post_zeros) w.add_bits(0, s.post_zeros);
    return true;
}

template <int MOD, class W>
R4_HD void slice_loop(PulseView const &p, SlicerParams const &t, W &w)
{
    SlicerState st;
    if (!slicer_begin<MOD>(p, t, st)) return;
    while (st.k < st.total || st.pending) {
        Step s = slicer_step<MOD>(p, t, st);
        if (!slicer_apply(s, w)) break;
    }
}

template <class W>
R4_HD void slice_dispatch(PulseView const &p, SlicerParams const &t, W &w)
{
    // the four slicers that carry 97 % of the reference's devices get their own loop
    switch (t.modulation) {
    case kModOokPwm: case kModFskPwm: slice_loop<kModOokPwm>(p, t, w); return;
    case kModOokPpm: slice_loop<kModOokPpm>(p, t, w); return;
    case kModOokPcm: case kModFskPcm: slice_loop<kModOokPcm>(p, t, w); return;
    case kModOokMc: case kModFskMc: slice_loop<kModOokMc>(p, t, w); return;
    default: break;
    }
    slice_loop<kModAny>(p, t, w);
}

} // namespace r433b
