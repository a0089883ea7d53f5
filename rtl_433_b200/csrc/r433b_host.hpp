// r433b_host.hpp -- host-only helpers shared by the C ABI (r433b_api.cu) and the CPU unit-test
// driver (tests/host_core.cpp): the float/double parameter derivations the reference does once
// per run, and the decoder-side re-inflation of compact events into a bitbuffer_t.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/r433b.h"
#include "../../include/r433b_abi.h"
#include "r433b_core.cuh"
#include "r433b_slice.cuh"

namespace r433b {

// include/baseband.h:43-46 with _exp10f(x) = powf(10, x); src/pulse_detect.c:86-98, :24
inline Levels compute_levels(int use_mag, float level_limit, float min_level, float min_snr)
{
    Levels lv;
    if (use_mag) {
        lv.fixed_high = level_limit < 0.0 ? (int)(powf(10, (level_limit + 84.2884f) / 20.0f)) : 0;
        lv.min_high = (int)(powf(10, (min_level + 84.2884f) / 20.0f));
        lv.ratio = (int)(0.5 + powf(10, min_snr / 20.0f));
    } else {
        lv.fixed_high = level_limit < 0.0 ? (int)(powf(10, (level_limit + 42.1442f) / 10.0f)) : 0;
        lv.min_high = (int)(powf(10, (min_level + 42.1442f) / 10.0f));
        lv.ratio = (int)(0.5 + powf(10, min_snr / 10.0f));
    }
    lv.max_high = (int)(powf(10, (0 + 42.1442f) / 10.0f));
    return lv;
}

// src/baseband.c:217-231 (cu8) and :310-324 (cs16): double arithmetic, truncation to int
inline void fm_coeffs(int cs16, uint32_t rate, float low_pass, int &a1, int &b0)
{
    if (low_pass > 1e4f)
        low_pass = low_pass / rate;
    else if (low_pass >= 1.0f)
        low_pass = 1e6f / low_pass / rate;
    double ita = 1.0 / tan(M_PI_2 * low_pass);
    if (!cs16) {
        double gain = 1.0 / (1.0 + ita) / 2;
        a1 = (int)((ita - 1.0) * gain * 32768);
        b0 = (int)(gain * 32768);
    } else {
        double gain = 1.0 / (1.0 + ita);
        a1 = (int)((ita - 1.0) * gain * (1 << 30));
        b0 = (int)(gain * (1 << 30));
    }
}

// the preamble shared by all slicers (e.g. src/pulse_slicer.c:341-359), evaluated here on the
// host in float exactly as the reference does, so the device only sees integers
inline SlicerParams scale_device(r433b_device const &d, uint32_t rate)
{
    SlicerParams t{};
    float per_us = rate / 1.0e6f;
    t.modulation = (int)d.modulation;
    t.s_short = d.short_width * per_us;
    t.s_long = d.long_width * per_us;
    t.s_reset = d.reset_limit * per_us;
    t.s_gap = d.gap_limit * per_us;
    t.s_sync = d.sync_width * per_us;
    t.s_tol = d.tolerance * per_us;
    bool bad3 = (d.short_width > 0 && t.s_short <= 0) || (d.long_width > 0 && t.s_long <= 0)
            || (d.reset_limit > 0 && t.s_reset <= 0);
    bool bad6 = bad3 || (d.gap_limit > 0 && t.s_gap <= 0) || (d.sync_width > 0 && t.s_sync <= 0)
            || (d.tolerance > 0 && t.s_tol <= 0);
    t.ok = (bad6 ? 0 : 1) | (bad3 ? 0 : 2);
    if ((int)d.modulation == kModOokRzi) { // src/pulse_slicer.c:870-873: only three widths are scaled
        t.s_gap = t.s_sync = t.s_tol = 0;
    }
    t.f_short = d.short_width > 0.0f ? 1.0f / (d.short_width * per_us) : 0;
    t.f_long = d.long_width > 0.0f ? 1.0f / (d.long_width * per_us) : 0;
    t.priority = d.priority;
    return t;
}


// The device list k_slice2 walks for one package type (1 = OOK, 2 = FSK): each device
// run_ook_demods / run_fsk_demods hand such a package to (src/r_api.c:438-550), once, as an index
// into `devs`.  k_slice2's work items are device major, and the warps of the GPU fetch them in list
// order, so the devices next to each other in the list are the ones that run side by side: sorted by
// modulation, most warps of the GPU run the same slicer code at any moment (instruction cache); within
// a modulation, reset limit and short width put devices of similar timing next to each other.
inline std::vector<unsigned> slice_list(std::vector<r433b_device> const &devs, int package_type)
{
    std::vector<unsigned> v;
    for (unsigned i = 0; i < (unsigned)devs.size(); ++i)
        if (device_takes((int)devs[i].modulation, package_type)) v.push_back(i);
    std::sort(v.begin(), v.end(), [&](unsigned a, unsigned c) {
        r433b_device const &x = devs[a], &y = devs[c];
        if (x.modulation != y.modulation) return x.modulation < y.modulation;
        if (x.reset_limit != y.reset_limit) return x.reset_limit < y.reset_limit;
        if (x.short_width != y.short_width) return x.short_width < y.short_width;
        return a < c;
    });
    return v;
}


// The header of an event of the wire format (r433b_slice.cuh); len = the event's words.
struct EventHead {
    uint32_t num_rows, dirty, free_row, len;
};

inline EventHead event_head(uint32_t h)
{
    if ((h & 0xff) == 0xff) return {1, 0, 1, 1}; // one-word event
    return {h & 0x7f, (h >> 7) & 1, (h >> 8) & 0xff, h >> 16};
}

// The rows of the event at ev (len words, head e), each as in the long form whatever form it is stored in:
// row(r, bits, syncs, data, words) with `words` data words at `data`.  Returns the offset of the first word after the
// rows (the dirty trailer, if any), or -1 if the event is malformed.
template <class Row>
inline int event_rows(uint32_t const *ev, EventHead const &e, Row &&row)
{
    uint32_t const end = e.len;
    uint32_t const h = ev[0];
    if ((h & 0xff) == 0xff) {
        uint32_t const data = h >> 16, bits = (h >> 8) & 31;
        if (bits > 16) return -1;
        row(0u, bits, (h >> 13) & 7, &data, bits ? 1u : 0u);
        return 1;
    }
    uint32_t q = 1;
    for (uint32_t r = 0; r < e.num_rows && r < R433B_BITBUF_ROWS; ++r) {
        if (q + 1 > end) return -1;
        uint32_t const w = ev[q];
        q += 1;
        if (w >> 31) { // short row
            uint32_t const data = w & 0xffff, bits = (w >> 16) & 31;
            if (bits > 16) return -1;
            row(r, bits, (w >> 21) & 0x3ff, &data, bits ? 1u : 0u);
            continue;
        }
        uint32_t const bits = w & 0xffff;
        uint32_t words = (bits + 31) / 32;
        if (e.dirty && r + 1 == e.num_rows) words = ev[end - 1];
        if (q + words > end) return -1;
        row(r, bits, w >> 16, ev + q, words);
        q += words;
    }
    return (int)q;
}

// One event of a pair's byte stream back into the decoder-facing struct
// (include/bitbuffer.h:34-40).  Row r's bytes go to bb + r*128 and may run on into the
// following rows exactly as the reference's spill-over does (src/bitbuffer.c:39-54).
inline int event_to_bitbuffer(uint8_t const *ev8, uint32_t pair_bytes, uint32_t index, struct bitbuffer *out,
        uint32_t *consumed)
{
    if (!ev8 || !out || (pair_bytes & 3)) return -1;
    uint32_t const *ev = reinterpret_cast<uint32_t const *>(ev8);
    uint32_t const total = pair_bytes / 4;
    uint32_t pos = 0;
    EventHead e;
    for (uint32_t i = 0;; ++i) {
        if (pos + 1 > total) return -1;
        e = event_head(ev[pos]);
        if (e.len < 1 || pos + e.len > total) return -1;
        if (i == index) break;
        pos += e.len;
    }
    memset(out, 0, sizeof(*out));
    out->num_rows = (uint16_t)e.num_rows;
    out->free_row = (uint16_t)e.free_row;
    uint8_t *flat = &out->bb[0][0];
    int const rc = event_rows(ev + pos, e, [&](uint32_t r, uint32_t bits, uint32_t syncs, uint32_t const *data, uint32_t words) {
        out->bits_per_row[r] = (uint16_t)bits;
        out->syncs_before_row[r] = (uint16_t)syncs;
        size_t at = (size_t)r * R433B_BITBUF_COLS;
        size_t room = sizeof(out->bb) - at;
        size_t nb = (size_t)words * 4;
        memcpy(flat + at, data, nb < room ? nb : room);
    });
    if (rc < 0) return -1;
    if (consumed) *consumed = (pos + e.len) * 4;
    return 0;
}

// The event at ev (head e) appended to `out` in the long form, the only one before one-word rows and events: a
// header, then every row as a header word and ceil(bits/32) data words, then the dirty trailer.  Returns -1 if the
// event is malformed.
inline int event_long_form(uint32_t const *ev, EventHead const &e, std::vector<uint32_t> &out)
{
    size_t const at = out.size();
    out.push_back(0);
    int const q = event_rows(ev, e, [&](uint32_t, uint32_t bits, uint32_t syncs, uint32_t const *data, uint32_t words) {
        out.push_back(bits | (syncs << 16));
        out.insert(out.end(), data, data + words);
    });
    if (q < 0) return -1;
    out.insert(out.end(), ev + q, ev + e.len);
    out[at] = e.num_rows | (e.dirty << 7) | (e.free_row << 8) | ((uint32_t)(out.size() - at) << 16);
    return 0;
}

} // namespace r433b
