// r433b_analyze_host.hpp -- the O(1) tail of the pulse analyzer on the host: from the five histograms k_analyze
// built for a package to the guessed modulation / flex-decoder timings, the RfRaw rendering and the text
// `rtl_433 -A` prints (src/pulse_analyzer.c:325-560).  The float and double expressions are the reference's.
#pragma once
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/r433b.h"
#include "../../include/r433b_abi.h"
#include "r433b_analyze.cuh"
#include "r433b_pulses.hpp"

namespace r433b {

// histogram_sort_mean / histogram_sort_count, src/pulse_analyzer.c:96-125: the reference's exchange sort
// (not stable, so the exact swap sequence matters when keys tie)
template <class Less>
inline void hist_exchange_sort(Histogram &h, Less less)
{
    if (h.bins_count < 2) return;
    for (unsigned n = 0; n + 1 < h.bins_count; ++n)
        for (unsigned m = n + 1; m < h.bins_count; ++m)
            if (less(h.bins[m], h.bins[n])) {
                HistBin t = h.bins[m];
                h.bins[m] = h.bins[n];
                h.bins[n] = t;
            }
}

inline int hist_find(Histogram const &h, int width) // histogram_find_bin_index, :156-164
{
    for (unsigned n = 0; n < h.bins_count; ++n)
        if (h.bins[n].min <= width && width <= h.bins[n].max) return (int)n;
    return -1;
}

inline void hist_print(TextOut &o, Histogram const &h, uint32_t rate) // histogram_print, :167-177
{
    for (unsigned n = 0; n < h.bins_count; ++n)
        o.put(" [%2u] count: %4u,  width: %4.0f us [%.0f;%.0f]\t(%4i S)\n", n, h.bins[n].count, h.bins[n].mean * 1e6 / rate,
                h.bins[n].min * 1e6 / rate, h.bins[n].max * 1e6 / rate, h.bins[n].mean);
}

// the 1024-byte hex builder of :179-209
struct HexBuilder {
    uint8_t p[1024];
    unsigned idx = 0;
    void byte(uint8_t v)
    {
        if (idx < sizeof(p)) p[idx++] = v;
    }
    void word(uint16_t v)
    {
        if (idx + 1 < sizeof(p)) {
            p[idx++] = v >> 8;
            p[idx++] = v & 0xff;
        }
    }
    void print(TextOut &o) const
    {
        for (unsigned i = 0; i < idx; ++i) o.put("%02X", p[i]);
    }
};

// pulse_analyzer_check(), src/pulse_analyzer.c:214-276, from the same histograms: 1 when the package has more than
// one pulse and more than a single pulse width and gap width (the zero-width FSK bin left out), else 0.
inline int analysis_check(unsigned num_pulses, r433b_analysis const &an)
{
    if (num_pulses <= 1) return 0;
    Histogram pulses = an.hist[0];
    hist_exchange_sort(pulses, [](HistBin const &a, HistBin const &b) { return a.mean < b.mean; });
    if (pulses.bins[0].mean == 0) hist_delete(pulses, 0);
    return pulses.bins_count == 1 && an.hist[1].bins_count == 1 ? 0 : 1;
}

// What the analyzer concludes for one package.  `pd` must hold the package as the analyzer sees it (levels and
// estimates filled in); `type` is PULSE_DATA_OOK / _FSK (1 / 2).  Returns the text; fills guess / last_gap.
inline size_t analysis_finish(struct pulse_data const *pd, int type, r433b_analysis const &an, r433b_guess *guess, char *buf, size_t cap)
{
    TextOut o{buf, cap};
    r433b_guess g{};
    g.last_gap = -1;
    if (pd->num_pulses == 0) {
        o.put("No pulses detected.\n");
        if (guess) *guess = g;
        return o.len;
    }
    double const to_ms = 1e3 / pd->sample_rate;
    double const to_us = 1e6 / pd->sample_rate;
    Histogram pulses = an.hist[0], gaps = an.hist[1];
    Histogram const &periods_pg = an.hist[2], &periods_gp = an.hist[3], &timings = an.hist[4];

    o.put("Analyzing pulses...\n");
    o.put("Total count: %4u,  width: %4.2f ms\t\t(%5i S)\n", pd->num_pulses, an.total_period * to_ms, an.total_period);
    o.put("Pulse width distribution:\n");
    hist_print(o, pulses, pd->sample_rate);
    o.put("Gap width distribution:\n");
    hist_print(o, gaps, pd->sample_rate);
    o.put("Pulse+gap period distribution:\n");
    hist_print(o, periods_pg, pd->sample_rate);
    o.put("Gap+pulse period distribution:\n");
    hist_print(o, periods_gp, pd->sample_rate);
    o.put("Timing distribution:\n");
    hist_print(o, timings, pd->sample_rate);
    o.put("Level estimates [high, low]: %6i, %6i\n", pd->ook_high_estimate, pd->ook_low_estimate);
    o.put("RSSI: %.1f dB SNR: %.1f dB Noise: %.1f dB\n", pd->rssi_db, pd->snr_db, pd->noise_db);
    o.put("Frequency offsets [F1, F2]:  %6i, %6i\t(%+.1f kHz, %+.1f kHz)\n", pd->fsk_f1_est, pd->fsk_f2_est,
            ((float)pd->fsk_f1_est / INT16_MAX) * (pd->sample_rate / 2.0 / 1000.0),
            ((float)pd->fsk_f2_est / INT16_MAX) * (pd->sample_rate / 2.0 / 1000.0));

    o.put("Guessing modulation: ");
    hist_exchange_sort(pulses, [](HistBin const &a, HistBin const &b) { return a.mean < b.mean; });
    hist_exchange_sort(gaps, [](HistBin const &a, HistBin const &b) { return a.mean < b.mean; });
    if (pulses.bins[0].mean == 0) hist_delete(pulses, 0); // the FSK initial zero-bin

    bool const fsk = type == 2;
    unsigned const np = pulses.bins_count, ng = gaps.bins_count;
    HistBin const *pb = pulses.bins, *gb = gaps.bins;
    auto top_gap_limit = [&]() { return (float)(to_us * (gb[ng - 1].max + 1)); }; // "above biggest gap"; ng - 1 wraps like the reference's index
    auto near = [&](int v, int target) {
        int d = v - target;
        if (d < 0) d = -d;
        return d <= pb[0].mean / 8;
    };
    if (pd->num_pulses == 1) {
        o.put("Single pulse detected. Probably Frequency Shift Keying or just noise...\n");
    } else if (np == 1 && ng == 1) {
        o.put("Un-modulated signal. Maybe a preamble...\n");
    } else if (np == 1 && ng > 1) {
        o.put("Pulse Position Modulation with fixed pulse width\n");
        g.modulation = kModOokPpm;
        g.short_width = (float)(to_us * gb[0].mean);
        g.long_width = (float)(to_us * gb[1].mean);
        g.gap_limit = (float)(to_us * (gb[1].max + 1));
        g.reset_limit = top_gap_limit();
    } else if (np == 2 && ng == 1) {
        o.put("Pulse Width Modulation with fixed gap\n");
        g.modulation = fsk ? kModFskPwm : kModOokPwm;
        g.short_width = (float)(to_us * pb[0].mean);
        g.long_width = (float)(to_us * pb[1].mean);
        g.tolerance = (float)((g.long_width - g.short_width) * 0.4);
        g.reset_limit = top_gap_limit();
    } else if (np == 2 && ng == 2 && periods_pg.bins_count == 1) {
        o.put("Pulse Width Modulation with fixed period\n");
        g.modulation = fsk ? kModFskPwm : kModOokPwm;
        g.short_width = (float)(to_us * pb[0].mean);
        g.long_width = (float)(to_us * pb[1].mean);
        g.tolerance = (float)((g.long_width - g.short_width) * 0.4);
        g.reset_limit = top_gap_limit();
    } else if (np == 2 && ng == 2 && periods_pg.bins_count == 3) {
        o.put("Manchester coding\n");
        g.modulation = fsk ? kModFskMc : kModOokMc;
        g.short_width = (float)(to_us * (pb[0].mean < pb[1].mean ? pb[0].mean : pb[1].mean));
        g.long_width = 0;
        g.reset_limit = top_gap_limit();
    } else if (np == 2 && ng >= 3) {
        o.put("Pulse Width Modulation with multiple packets\n");
        g.modulation = fsk ? kModFskPwm : kModOokPwm;
        g.short_width = (float)(to_us * pb[0].mean);
        g.long_width = (float)(to_us * pb[1].mean);
        g.gap_limit = (float)(to_us * (gb[1].max + 1));
        g.tolerance = (float)((g.long_width - g.short_width) * 0.4);
        g.reset_limit = top_gap_limit();
    } else if (np >= 3 && ng >= 3 && near(pb[1].mean, 2 * pb[0].mean) && near(pb[2].mean, 3 * pb[0].mean)
            && near(gb[0].mean, pb[0].mean) && near(gb[1].mean, 2 * pb[0].mean) && near(gb[2].mean, 3 * pb[0].mean)) {
        o.put("Non Return to Zero coding (Pulse Code)\n");
        g.modulation = fsk ? kModFskPcm : kModOokPcm;
        g.short_width = (float)(to_us * pb[0].mean);
        g.long_width = (float)(to_us * pb[0].mean);
        g.reset_limit = (float)(to_us * pb[0].mean * 1024);
    } else if (np == 3) {
        o.put("Pulse Width Modulation with sync/delimiter\n");
        // the rarest pulse width is taken for the delimiter
        hist_exchange_sort(pulses, [](HistBin const &a, HistBin const &b) { return a.count < b.count; });
        int const p1 = pb[1].mean, p2 = pb[2].mean;
        g.modulation = fsk ? kModFskPwm : kModOokPwm;
        g.short_width = (float)(to_us * (p1 < p2 ? p1 : p2));
        g.long_width = (float)(to_us * (p1 < p2 ? p2 : p1));
        g.sync_width = (float)(to_us * pb[0].mean);
        g.reset_limit = top_gap_limit();
    } else {
        o.put("No clue...\n");
    }

    // RfRaw line, :461-543
    bool impossible = false;
    if (timings.bins_count <= 8) {
        auto push_bins = [&](HexBuilder &h) {
            for (unsigned b = 0; b < timings.bins_count; ++b) {
                double w = timings.bins[b].mean * to_us;
                if (w < 0) w = 0;
                h.word(w < USHRT_MAX ? (uint16_t)w : (uint16_t)USHRT_MAX);
            }
        };
        auto code_of = [&](unsigned i, HexBuilder &h) {
            int const p = hist_find(timings, pd->pulse[i]), gi = hist_find(timings, pd->gap[i]);
            if (p < 0 || gi < 0) return false;
            h.byte((uint8_t)(0x80 | (p << 4) | gi));
            return true;
        };
        if (gaps.bins_count <= 2) { // one long B1 code
            HexBuilder h;
            h.byte(0xaa);
            h.byte(0xb1);
            h.byte((uint8_t)timings.bins_count);
            push_bins(h);
            for (unsigned i = 0; i < pd->num_pulses && !impossible; ++i)
                if (!code_of(i, h)) impossible = true;
            if (!impossible) {
                h.byte(0x55);
                o.put("view at https://triq.org/pdv/#");
                h.print(o);
                o.put("\n");
            }
        } else { // B0 codes, cut at the gaps of the 4th-longest class or longer
            unsigned const limit_bin = gaps.bins_count - 1 < 3 ? gaps.bins_count - 1 : 3;
            int const limit = gaps.bins[limit_bin].min;
            static thread_local HexBuilder hs[32];
            for (auto &h : hs) {
                h.idx = 0;
                memset(h.p, 0, sizeof(h.p));
            }
            unsigned cnt = 0, i = 0;
            while (i < pd->num_pulses && cnt < 32 && !impossible) {
                HexBuilder &h = hs[cnt];
                h.byte(0xaa);
                h.byte(0xb0);
                h.byte(0); // length, patched below
                h.byte((uint8_t)timings.bins_count);
                h.byte(1); // repeats
                push_bins(h);
                for (; i < pd->num_pulses; ++i) {
                    if (!code_of(i, h)) {
                        impossible = true;
                        break;
                    }
                    if (pd->gap[i] >= limit) {
                        ++i;
                        break;
                    }
                }
                if (impossible) break;
                h.byte(0x55);
                h.p[2] = h.idx - 4 <= 255 ? (uint8_t)(h.idx - 4) : 0;
                if (cnt > 0 && hs[cnt - 1].idx == h.idx && !memcmp(&hs[cnt - 1].p[5], &h.p[5], h.idx - 5)) {
                    h.idx = 0;            // same as the group before:
                    hs[cnt - 1].p[4] += 1; // one more repeat of it
                } else {
                    cnt++;
                }
            }
            if (!impossible) {
                o.put("view at https://triq.org/pdv/#");
                for (unsigned j = 0; j < cnt; ++j) {
                    if (j > 0) o.put("+");
                    hs[j].print(o);
                }
                o.put("\n");
                if (cnt >= 32) o.put("Too many pulse groups (%u pulses missed in rfraw)\n", pd->num_pulses - i);
            }
        }
    }
    if (impossible) {
        // A width that fell out of a full (16-bin) histogram lies in no bin: the reference prints this and exit(1)s.
        o.put("pulse_analyzer: this can't happen\n");
        g.modulation = 0;
        if (guess) *guess = g;
        return o.len;
    }

    // trial demodulation, :545-557: the text here, the slicer run on the GPU (k_slice_own)
    if (g.modulation) {
        o.put("Attempting demodulation... short_width: %.0f, long_width: %.0f, reset_limit: %.0f, sync_width: %.0f\n",
                g.short_width, g.long_width, g.reset_limit, g.sync_width);
        int const terminated = (int)(g.reset_limit / to_us + 1); // "Be sure to terminate package"
        switch (g.modulation) {
        case kModFskPcm:
            o.put("Use a flex decoder with -X 'n=name,m=FSK_PCM,s=%.0f,l=%.0f,r=%.0f'\n", g.short_width, g.long_width, g.reset_limit);
            break;
        case kModOokPpm:
            o.put("Use a flex decoder with -X 'n=name,m=OOK_PPM,s=%.0f,l=%.0f,g=%.0f,r=%.0f'\n", g.short_width, g.long_width,
                    g.gap_limit, g.reset_limit);
            g.last_gap = terminated;
            break;
        case kModOokPwm:
            o.put("Use a flex decoder with -X 'n=name,m=OOK_PWM,s=%.0f,l=%.0f,r=%.0f,g=%.0f,t=%.0f,y=%.0f'\n", g.short_width,
                    g.long_width, g.reset_limit, g.gap_limit, g.tolerance, g.sync_width);
            g.last_gap = terminated;
            break;
        case kModFskPwm:
            o.put("Use a flex decoder with -X 'n=name,m=FSK_PWM,s=%.0f,l=%.0f,r=%.0f,g=%.0f,t=%.0f,y=%.0f'\n", g.short_width,
                    g.long_width, g.reset_limit, g.gap_limit, g.tolerance, g.sync_width);
            g.last_gap = terminated;
            break;
        case kModOokMc:
            o.put("Use a flex decoder with -X 'n=name,m=OOK_MC_ZEROBIT,s=%.0f,l=%.0f,r=%.0f'\n", g.short_width, g.long_width, g.reset_limit);
            g.last_gap = terminated;
            break;
        default: // OOK_PCM and FSK_MC_ZEROBIT guesses have no slicer call in the reference
            o.put("Unsupported\n");
            g.sliced = 0;
            break;
        }
        g.sliced = g.modulation == kModFskPcm || g.last_gap >= 0;
    }
    o.put("\n");
    if (guess) *guess = g;
    return o.len;
}

} // namespace r433b
