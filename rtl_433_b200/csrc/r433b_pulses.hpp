// r433b_pulses.hpp -- pulse-level I/O around the slicers (SURVEY 8(f4)): the text formats the reference
// reads and writes packages in, on the host.
//
//   reading:  `.ook` pulse files          pulse_data_load()          src/pulse_data.c:123-181
//             RfRaw B0/B1 hex lines       rfraw_check / rfraw_parse  src/rfraw.c:67-206
//   writing:  `.ook`                      pulse_data_dump()          src/pulse_data.c:193-226
//             VCD                         pulse_data_print_vcd()     src/pulse_data.c:102-121
//             logic.u8                    pulse_data_dump_raw()      src/pulse_data.c:58-68
//
// A loaded set of packages goes to the GPU through r433b_process_pulses() (the slicer stage only): the same slicers,
// the same event arena, the same replay as packages that came out of k_detect.  Host-only, no CUDA here.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/r433b_abi.h"

namespace r433b {

// ---------------------------------------------------------------------------- RfRaw ----------

// A cursor over hex text; blanks, tabs, '-' and ':' between digits are skipped (src/rfraw.c:16-36).
struct HexCursor {
    char const *p;

    int nibble()
    {
        if (!p || !*p) return -1;
        while (*p == ' ' || *p == '\t' || *p == '-' || *p == ':') ++p;
        char c = *p;
        int v = c >= '0' && c <= '9' ? c - '0' : c >= 'A' && c <= 'F' ? c - 'A' + 10 : c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1;
        if (v >= 0) ++p;
        return v;
    }
    int byte()
    {
        int h = nibble(), l = nibble();
        return h >= 0 && l >= 0 ? (h << 4) | l : -1;
    }
    int word()
    {
        int h = byte(), l = byte();
        return h >= 0 && l >= 0 ? (h << 8) | l : -1;
    }
};

// "AA B0" or "AA B1" in front (src/rfraw.c:67-74)
inline bool rfraw_is(char const *text)
{
    HexCursor c{text};
    if (c.nibble() != 0xa || c.nibble() != 0xa || c.nibble() != 0xb) return false;
    return (c.nibble() | 1) == 1;
}

// One AA B0 / AA B1 group appended to `d` (src/rfraw.c:96-184).  Returns false when the text is not a group.
inline bool rfraw_group(struct pulse_data *d, HexCursor &c)
{
    if (!c.p || !*c.p) return false;
    if (c.byte() != 0xaa) return false;
    int const fmt = c.byte();
    if (fmt != 0xb0 && fmt != 0xb1) return false;
    if (fmt == 0xb0) c.byte(); // length, unused
    int const n_bins = c.byte();
    if (n_bins > 8) return false;
    int repeats = 1;
    if (fmt == 0xb0) repeats = c.byte();
    int bins[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n_bins; ++i) bins[i] = c.word();

    // old format: one nibble per width, pulses and gaps alternating; new: bit 3 of a nibble marks a pulse
    bool old_format = true;
    for (HexCursor t{c.p}; *t.p;) {
        int b = t.byte();
        if (b < 0 || b == 0x55) break;
        if (b & 0x88) {
            old_format = false;
            break;
        }
    }

    unsigned const first = d->num_pulses;
    bool want_pulse = true, at_byte = true;
    // The reference's loop condition tests the cursor POINTER (`while (*p)` on a char const **), so the loop only
    // ends at the 0x55 marker, at a full array, or -- without a marker -- by failing on the end of the text:
    // then the group is not finished (no repeats, sample rate untouched), the widths read so far stay.
    for (;;) {
        if (at_byte) {
            HexCursor peek{c.p};
            if (peek.byte() == 0x55) { // end marker
                c.byte();
                break;
            }
        }
        int const w = c.nibble();
        at_byte = !at_byte;
        if (w < 0) return false;
        if (w >= 8 || (old_format && !at_byte)) { // a pulse width
            if (!want_pulse) { // two pulses in a row: an empty gap between them
                d->gap[d->num_pulses] = 0;
                d->num_pulses++;
            }
            d->pulse[d->num_pulses] = bins[w & 7];
            want_pulse = false;
        } else { // a gap width
            if (want_pulse) d->pulse[d->num_pulses] = 0;
            d->gap[d->num_pulses] = bins[w];
            d->num_pulses++;
            want_pulse = true;
        }
        if (d->num_pulses >= R433B_PD_MAX_PULSES) break;
    }
    unsigned const n = d->num_pulses - first;
    for (int r = 1; r < repeats && d->num_pulses + n <= R433B_PD_MAX_PULSES; ++r) {
        memcpy(&d->pulse[d->num_pulses], &d->pulse[first], n * sizeof(int));
        memcpy(&d->gap[d->num_pulses], &d->gap[first], n * sizeof(int));
        d->num_pulses += n;
    }
    d->sample_rate = 1000000; // RfRaw widths are microseconds
    return true;
}

// All groups of a line ('+', blanks, line ends between them), appended; `d` is not cleared (src/rfraw.c:186-206).
inline bool rfraw_append(struct pulse_data *d, char const *text)
{
    if (!text || !*text) return false;
    HexCursor c{text};
    while (*c.p) {
        while (*c.p == ' ' || *c.p == '\t' || *c.p == '\r' || *c.p == '\n' || *c.p == '+' || *c.p == '-') ++c.p;
        if (!rfraw_group(d, c)) break;
    }
    return true;
}

// ------------------------------------------------------------------------ .ook reader --------

// fgets() over a memory buffer: at most cap-1 characters, through the first '\n'.
struct TextReader {
    char const *p, *end;

    bool gets(char *s, int cap)
    {
        if (p >= end) return false;
        int n = 0;
        while (n < cap - 1 && p < end) {
            char ch = *p++;
            s[n++] = ch;
            if (ch == '\n') break;
        }
        s[n] = 0;
        return true;
    }
};

// One pulse_data_load() call: the next package of the text, or num_pulses == 0 at its end.  `line` is the
// caller's 1024-byte line buffer (the reference's `char s[1024]`): a last line without '\n' lets the second
// strtol() start one character past the terminator, i.e. in whatever an earlier, longer line left there.
inline void ook_load_next(TextReader &rd, uint32_t samp_rate, struct pulse_data *d, char *line)
{
    memset(d, 0, sizeof(*d));
    d->sample_rate = samp_rate;
    double const to_sample = samp_rate / 1e6;
    int i = 0;
    while (i < R433B_PD_MAX_PULSES && rd.gets(line, 1024)) {
        if (!strncmp(line, ";freq1", 6)) d->freq1_hz = strtol(line + 6, nullptr, 10);
        if (!strncmp(line, ";freq2", 6)) d->freq2_hz = strtol(line + 6, nullptr, 10);
        // ";received <time>" sets the reference's clock (demod->now); times are not part of this path
        if (line[0] == ';') {
            if (i) break; // the end marker, or the next package's header
            continue;     // still in the header
        }
        if (rfraw_is(line)) {
            rfraw_append(d, line);
            i = (int)d->num_pulses;
            continue;
        }
        char *endp = nullptr;
        long const mark = strtol(line, &endp, 10);
        long const space = strtol(endp < line + 1023 ? endp + 1 : endp, &endp, 10);
        if (mark < 0 || space < 0) continue;
        d->pulse[i] = (int)(to_sample * mark);
        d->gap[i++] = (int)(to_sample * space);
    }
    d->num_pulses = (unsigned)i;
}

// ---------------------------------------------------------------------------- writers --------

// snprintf-style appender that keeps counting when the buffer is full
struct TextOut {
    char *buf;
    size_t cap, len = 0;

    void put(char const *fmt, ...)
    {
        va_list ap;
        va_start(ap, fmt);
        int n = vsnprintf(len < cap ? buf + len : nullptr, len < cap ? cap - len : 0, fmt, ap);
        va_end(ap);
        if (n > 0) len += (size_t)n;
    }
};

// pulse_data_dump(), src/pulse_data.c:193-226.  `received`: the text after ";received " or nullptr to leave
// that line out (the reference prints the wall clock there).
inline size_t format_ook(struct pulse_data const *d, char const *received, char *buf, size_t cap)
{
    TextOut o{buf, cap};
    if (received) o.put(";received %s\n", received);
    if (d->fsk_f2_est) {
        o.put(";fsk %u pulses\n", d->num_pulses);
        o.put(";freq1 %.0f\n", d->freq1_hz);
        o.put(";freq2 %.0f\n", d->freq2_hz);
    } else {
        o.put(";ook %u pulses\n", d->num_pulses);
        o.put(";freq1 %.0f\n", d->freq1_hz);
    }
    o.put(";centerfreq %.0f Hz\n", d->centerfreq_hz);
    o.put(";samplerate %u Hz\n", d->sample_rate);
    o.put(";sampledepth %u bits\n", d->depth_bits);
    o.put(";range %.1f dB\n", d->range_db);
    o.put(";rssi %.1f dB\n", d->rssi_db);
    o.put(";snr %.1f dB\n", d->snr_db);
    o.put(";noise %.1f dB\n", d->noise_db);
    double const to_us = 1e6 / d->sample_rate;
    for (unsigned i = 0; i < d->num_pulses; ++i) o.put("%.0f %.0f\n", d->pulse[i] * to_us, d->gap[i] * to_us);
    o.put(";end\n");
    return o.len;
}

// pulse_data_print_pulse_header(), src/pulse_data.c:183-191 (`created`: text after ";created ", or nullptr)
inline size_t format_ook_header(char const *created, char *buf, size_t cap)
{
    TextOut o{buf, cap};
    o.put(";pulse data\n;version 1\n;timescale 1us\n");
    if (created) o.put(";created %s\n", created);
    return o.len;
}

// pulse_data_print_vcd(), src/pulse_data.c:102-121: ch_id '\'' for OOK (AM), '"' for FSK (FM).  The time
// scale is an INTEGER quotient kept in a float, and positions are multiplied in float -- as in the reference.
inline size_t format_vcd(struct pulse_data const *d, int ch_id, char *buf, size_t cap)
{
    TextOut o{buf, cap};
    float const scale = d->sample_rate <= 500000 ? (float)(1000000 / d->sample_rate) : (float)(10000000 / d->sample_rate);
    uint64_t pos = d->offset;
    for (unsigned n = 0; n < d->num_pulses; ++n) {
        if (n == 0)
            o.put("#%.f 1/ 1%c\n", (double)((float)pos * scale), ch_id);
        else
            o.put("#%.f 1%c\n", (double)((float)pos * scale), ch_id);
        pos += d->pulse[n];
        o.put("#%.f 0%c\n", (double)((float)pos * scale), ch_id);
        pos += d->gap[n];
    }
    if (d->num_pulses > 0) o.put("#%.f 0/\n", (double)((float)pos * scale));
    return o.len;
}

// pulse_data_print_vcd_header(), src/pulse_data.c:78-100 with nice_freq() of src/r_util.c:290-307
inline size_t format_vcd_header(uint32_t sample_rate, char const *date, char *buf, size_t cap)
{
    TextOut o{buf, cap};
    char freq[32];
    double const f = sample_rate;
    if (f >= 1e9) snprintf(freq, sizeof(freq), "%.3fGHz", f / 1e9);
    else if (f >= 1e6) snprintf(freq, sizeof(freq), "%.3fMHz", f / 1e6);
    else if (f >= 1e3) snprintf(freq, sizeof(freq), "%.3fkHz", f / 1e3);
    else snprintf(freq, sizeof(freq), "%f", f);
    o.put("$date %s $end\n", date ? date : "");
    o.put("$version rtl_433 0.1.0 $end\n");
    o.put("$comment Acquisition at %s Hz $end\n", freq);
    o.put("$timescale %s $end\n", sample_rate <= 500000 ? "1 us" : "100 ns");
    o.put("$scope module rtl_433 $end\n$var wire 1 / FRAME $end\n$var wire 1 ' AM $end\n$var wire 1 \" FM $end\n");
    o.put("$upscope $end\n$enddefinitions $end\n#0 0/ 0' 0\"\n");
    return o.len;
}

// pulse_data_dump_raw(), src/pulse_data.c:44-68: pulses as 0x01 | bits, gaps as 0x01, clipped to the buffer
inline void dump_logic_u8(uint8_t *buf, uint64_t len, uint64_t buf_offset, struct pulse_data const *d, uint8_t bits)
{
    int64_t pos = (int64_t)(d->offset - buf_offset);
    auto fill = [&](int value, int64_t at, int64_t n) {
        if (at < 0) {
            n += at;
            at = 0;
        }
        if (at + n > (int64_t)len) n = (int64_t)len - at;
        if (n > 0) memset(buf + at, value, (size_t)n);
    };
    for (unsigned n = 0; n < d->num_pulses; ++n) {
        fill(0x01 | bits, pos, d->pulse[n]);
        pos += d->pulse[n];
        fill(0x01, pos, d->gap[n]);
        pos += d->gap[n];
    }
}

// ------------------------------------------------------------------------- package set -------

// Packages waiting for r433b_process_pulses(): what the reference would hold in demod->pulse_data, one after
// the other.  Widths live in two pools; a package owns num_pulses + 1 entries (the entry after the last pulse
// is observable: pulse_slicer_osv1 reads it, an RfRaw line can leave a pulse without a gap there).
struct PulseSet {
    struct Meta {
        uint32_t stream, seq, rate, num_pulses, first, count;
        int32_t type;
        int32_t fsk_f1_est, fsk_f2_est;
        float freq1_hz, freq2_hz;
    };
    std::vector<Meta> pk;
    std::vector<int32_t> pulse, gap;
    std::vector<uint32_t> next_seq; // per stream

    void add(uint32_t stream, struct pulse_data const *d)
    {
        Meta m{};
        m.stream = stream;
        if (next_seq.size() <= stream) next_seq.resize((size_t)stream + 1, 0);
        m.seq = next_seq[stream]++;
        m.rate = d->sample_rate;
        m.num_pulses = d->num_pulses > R433B_PD_MAX_PULSES ? R433B_PD_MAX_PULSES : d->num_pulses;
        m.first = (uint32_t)pulse.size();
        m.count = m.num_pulses < R433B_PD_MAX_PULSES ? m.num_pulses + 1 : m.num_pulses;
        // run_ook_demods unless fsk_f2_est is set (src/rtl_433.c:1774-1778, :1626-1631)
        m.type = d->fsk_f2_est ? 2 : 1;
        m.fsk_f1_est = d->fsk_f1_est;
        m.fsk_f2_est = d->fsk_f2_est;
        m.freq1_hz = d->freq1_hz;
        m.freq2_hz = d->freq2_hz;
        pulse.insert(pulse.end(), d->pulse, d->pulse + m.count);
        gap.insert(gap.end(), d->gap, d->gap + m.count);
        pk.push_back(m);
    }

    void get(uint32_t i, struct pulse_data *d) const
    {
        Meta const &m = pk[i];
        memset(d, 0, sizeof(*d));
        d->sample_rate = m.rate;
        d->num_pulses = m.num_pulses;
        memcpy(d->pulse, pulse.data() + m.first, m.count * sizeof(int));
        memcpy(d->gap, gap.data() + m.first, m.count * sizeof(int));
        d->fsk_f1_est = m.fsk_f1_est;
        d->fsk_f2_est = m.fsk_f2_est;
        d->freq1_hz = m.freq1_hz;
        d->freq2_hz = m.freq2_hz;
    }
};

// The file loop of `rtl_433 -r x.ook` (src/rtl_433.c:1755-1760): pulse_data_load() until a package comes
// back empty.  Returns the number of packages appended for `stream`.
inline int load_ook_text(PulseSet &set, uint32_t stream, char const *text, size_t len, uint32_t samp_rate)
{
    TextReader rd{text, text + len};
    static thread_local struct pulse_data d;
    char line[1024];
    memset(line, 0, sizeof(line));
    int n = 0;
    for (;;) {
        ook_load_next(rd, samp_rate, &d, line);
        if (!d.num_pulses) break;
        set.add(stream, &d);
        n++;
    }
    return n;
}

} // namespace r433b
