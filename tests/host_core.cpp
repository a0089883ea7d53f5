// tests/host_core.cpp -- CPU unit-test driver for the __host__ __device__ building blocks of the
// product (rtl_433_b200/csrc/r433b_core.cuh, r433b_slice.cuh, r433b_host.hpp).
//
// TEST CODE ONLY.  It runs the same per-sample functions the sm_90a kernels call, one stream
// at a time and strictly sequentially, so their logic can be checked against the oracle on a
// machine without a GPU.  It is never built into, or reachable from, libr433b.so; the warp
// level orchestration of the kernels (bracket rounds, ballots) is covered by the -m gpu tests.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../rtl_433_b200/csrc/r433b_host.hpp"

using namespace r433b;

namespace {

struct HostCtx {
    int lane = 0;
    int nlanes = 1;
    void sync() {}
};

// same layouts as oracle/ref_harness.c so tests read all three with one reader
struct hc_package {
    int32_t type;
    int32_t block;
    uint64_t offset;
    uint32_t sample_rate, depth_bits, start_ago, end_ago, num_pulses;
    int32_t ook_low_estimate, ook_high_estimate, fsk_f1_est, fsk_f2_est;
    float freq1_hz, freq2_hz, centerfreq_hz, range_db, rssi_db, snr_db, noise_db;
    float sample_file_pos;
    uint32_t pulse_off, pulse_count;
    uint32_t first_event, num_events;
};

struct hc_event {
    uint32_t package;
    uint32_t dev;
    int32_t ret;
    uint32_t bb_idx;
    uint64_t hash;
};

uint64_t fnv1a(void const *p, size_t n)
{
    uint8_t const *b = (uint8_t const *)p;
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; ++i) {
        h ^= b[i];
        h *= 1099511628211ull;
    }
    return h;
}

struct Hc {
    int use_mag = 0;
    float level_limit = 0.0f, min_level = -12.1442f, min_snr = 9.0f, fm_low_pass = 0.0f;
    std::vector<r433b_device> devs;
    int store_bitbuffers = 1, store_stages = 0;
    std::vector<hc_package> pkgs;
    std::vector<hc_event> evts;
    std::vector<bitbuffer> bbs;
    std::vector<int32_t> ppool, gpool;
    std::vector<int16_t> am, fm;
};

void slice_package(Hc &h, int type, uint32_t rate, int const *pulse, int const *gap, unsigned n)
{
    PulseView pv{pulse, gap, n};
    unsigned next = 0;
    for (unsigned prio = 0; prio < 0xffffffffu; prio = next) {
        next = 0xffffffffu;
        for (size_t i = 0; i < h.devs.size(); ++i) {
            unsigned dp = h.devs[i].priority;
            if (dp > prio && dp < next) next = dp;
            if (dp != prio) continue;
            if (!device_takes((int)h.devs[i].modulation, type)) continue;
            SlicerParams sp = scale_device(h.devs[i], rate);
            EventWriter cw;
            cw.init(nullptr);
            slice_dispatch(pv, sp, cw);
            std::vector<uint32_t> buf(cw.committed + 2, 0xAAAAAAAAu);
            EventWriter sw;
            sw.init(buf.data(), cw.committed);
            slice_dispatch(pv, sp, sw);
            for (unsigned g = cw.committed; g < cw.committed + 2; ++g)
                if (buf[g] != 0xAAAAAAAAu) {
                    fprintf(stderr, "host_core: store pass wrote past its region (dev %zu)\n", i);
                    abort();
                }
            if (sw.committed != cw.committed || sw.events != cw.events) {
                fprintf(stderr, "host_core: count/store mismatch dev %zu: %u/%u bytes %u/%u events\n", i, cw.committed,
                        sw.committed, cw.events, sw.events);
                abort();
            }
            uint32_t at = 0;
            for (unsigned e = 0; e < sw.events; ++e) {
                bitbuffer bb;
                uint32_t used = 0;
                if (event_to_bitbuffer((uint8_t const *)buf.data() + at, sw.committed * 4 - at, 0, &bb, &used)) {
                    fprintf(stderr, "host_core: corrupt event stream\n");
                    abort();
                }
                at += used;
                hc_event ev;
                ev.package = h.pkgs.empty() ? 0xffffffffu : (uint32_t)(h.pkgs.size() - 1);
                ev.dev = (uint32_t)i;
                ev.ret = 0;
                ev.hash = fnv1a(&bb, sizeof(bb));
                ev.bb_idx = 0xffffffffu;
                if (h.store_bitbuffers) {
                    ev.bb_idx = (uint32_t)h.bbs.size();
                    h.bbs.push_back(bb);
                }
                h.evts.push_back(ev);
                if (!h.pkgs.empty()) h.pkgs.back().num_events++;
            }
        }
    }
}

} // namespace

extern "C" {

void *hc_create() { return new Hc(); }
void hc_destroy(void *p) { delete (Hc *)p; }
void hc_set_capture(void *p, int store_bitbuffers, int store_stages)
{
    ((Hc *)p)->store_bitbuffers = store_bitbuffers;
    ((Hc *)p)->store_stages = store_stages;
}
void hc_set_levels(void *p, int use_mag, float level_limit, float min_level, float min_snr)
{
    Hc *h = (Hc *)p;
    h->use_mag = use_mag;
    h->level_limit = level_limit;
    h->min_level = min_level;
    h->min_snr = min_snr;
}
void hc_set_fm_low_pass(void *p, float v) { ((Hc *)p)->fm_low_pass = v; }
int hc_add_device(void *p, r433b_device const *d)
{
    Hc *h = (Hc *)p;
    h->devs.push_back(*d);
    return (int)h->devs.size() - 1;
}

int hc_run_stream(void *p, void const *iq, size_t bytes, int SS, uint32_t rate, uint32_t center, int fpdm_mode,
        uint32_t block_bytes)
{
    Hc &h = *(Hc *)p;
    h.pkgs.clear();
    h.evts.clear();
    h.bbs.clear();
    h.ppool.clear();
    h.gpool.clear();
    h.am.clear();
    h.fm.clear();
    if (!block_bytes) block_bytes = 262144;
    unsigned const block = block_bytes / SS;
    unsigned long long const N = bytes / SS;
    unsigned long long const n_blocks = (N + block - 1) / block;
    Levels lv = compute_levels(h.use_mag, h.level_limit, h.min_level, h.min_snr);
    int fpdm = fpdm_mode == 2 ? (center > 800000000u ? 1 : 0) : fpdm_mode;
    int enable_fm = 0;
    for (auto const &d : h.devs)
        if (d.modulation >= 16) enable_fm = 1;
    int const a1 = ((int)(0.85408 * 32768)) >> 1, b0 = ((int)(0.07296 * 32768)) >> 1;
    int fa1 = 0, fb0 = 0;
    if (enable_fm) fm_coeffs(SS == 4, rate, h.fm_low_pass != 0.0f ? h.fm_low_pass : fpdm ? 0.2f : 0.1f, fa1, fb0);

    std::vector<int> scratch(4 * kMaxPulses, 0x5a5a5a5a); // deliberately dirty, like device scratch
    Trains tr{scratch.data(), scratch.data() + kMaxPulses, scratch.data() + 2 * kMaxPulses, scratch.data() + 3 * kMaxPulses};
    HostCtx cx;
    DetState d;
    det_reset(d);
    d.ook_hw = d.fsk_hw = kMaxPulses;
    int const per_ms = (int)(rate / 1000);
    int y_am = 0, y_fm = 0, x_prev = 0, xf_prev = 0, pr = 0, pq = 0;

    // a restatement of the package-emission arithmetic of k_detect (r433b_kernels.cuh, `emit`)
    auto emit = [&](int type, unsigned long long pos, bool flush) {
        PackageHeader ph = package_header(d, type);
        unsigned cnt = ph.num_pulses + 1 < (unsigned)kMaxPulses ? ph.num_pulses + 1 : (unsigned)kMaxPulses;
        unsigned long long blk = flush ? n_blocks : pos / block;
        unsigned long long bstart = blk * block;
        unsigned long long blen = flush ? 0 : (N - bstart < block ? N - bstart : block);
        hc_package k;
        memset(&k, 0, sizeof(k));
        k.type = type;
        k.block = (int)blk;
        k.offset = ph.offset;
        k.sample_rate = rate;
        k.start_ago = flush ? (unsigned)(N - ph.start_abs) : (unsigned)(bstart + blen - ph.start_abs);
        k.end_ago = flush ? 0u : (unsigned)(blen - (pos - bstart));
        k.num_pulses = ph.num_pulses;
        k.ook_low_estimate = ph.low;
        k.ook_high_estimate = ph.high;
        k.fsk_f1_est = ph.f1;
        k.fsk_f2_est = ph.f2;
        int const *sp = type == 1 ? tr.ook_pulse : tr.fsk_pulse;
        int const *sg = type == 1 ? tr.ook_gap : tr.fsk_gap;
        k.pulse_off = (uint32_t)h.ppool.size();
        k.pulse_count = cnt;
        h.ppool.insert(h.ppool.end(), sp, sp + cnt);
        h.gpool.insert(h.gpool.end(), sg, sg + cnt);
        k.first_event = (uint32_t)h.evts.size();
        h.pkgs.push_back(k);
        std::vector<int> pc(sp, sp + cnt), gc(sg, sg + cnt);
        slice_package(h, type, rate, pc.data(), gc.data(), ph.num_pulses);
    };

    uint8_t const *u8 = (uint8_t const *)iq;
    int16_t const *s16 = (int16_t const *)iq;
    for (unsigned long long n = 0; n < N;) {
        if (n % block == 0) det_call_boundary(d, lv);
        // sample maps + filters for sample n
        int ci, cq, x;
        if (SS == 2) {
            int ri = u8[2 * n], rq = u8[2 * n + 1];
            ci = ri - 128;
            cq = rq - 128;
            x = h.use_mag ? mag_cu8(ri, rq) : env_cu8(ri, rq);
        } else {
            ci = s16[2 * n];
            cq = s16[2 * n + 1];
            x = mag_cs16(ci, cq);
        }
        int xl = (n % block == 0) ? (int)(int16_t)x_prev : x_prev;
        y_am = iir16(y_am, a1, b0, x + xl);
        x_prev = x;
        int f;
        if (enable_fm) {
            if (SS == 2) {
                int xf = atan16(cq * pr - ci * pq, ci * pr + cq * pq);
                y_fm = iir16(y_fm, fa1, fb0, xf + xf_prev);
                xf_prev = xf;
                f = y_fm;
            } else {
                long long re = (long long)ci * pr + (long long)cq * pq;
                long long im = (long long)cq * pr - (long long)ci * pq;
                int xf = atan32((int)(unsigned)(unsigned long long)im, (int)(unsigned)(unsigned long long)re);
                y_fm = iir32(y_fm, fa1, fb0, (long long)xf + xf_prev);
                xf_prev = xf;
                f = y_fm >> 16;
            }
        } else {
            f = (int)(int16_t)x;
        }
        pr = ci;
        pq = cq;
        int a = (int)(int16_t)y_am;
        f = (int)(int16_t)f;
        if (h.store_stages) {
            h.am.push_back((int16_t)a);
            h.fm.push_back((int16_t)f);
        }
        // the detector may hand back the same sample after a package
        for (;;) {
            int ev = det_step(d, lv, tr, a, f, n, per_ms, fpdm, cx);
            if (!ev) break;
            emit(ev, n, false);
            det_call_boundary(d, lv);
        }
        ++n;
    }
    for (;;) {
        int ev = det_flush(d, tr, fpdm);
        if (!ev) break;
        emit(ev, N, true);
    }
    return (int)h.pkgs.size();
}

// run the slicers of the registered devices on a caller-built pulse train (slicer unit tests)
int hc_slice(void *p, int type, uint32_t rate, uint32_t n, int32_t const *pulse, int32_t const *gap)
{
    Hc &h = *(Hc *)p;
    h.pkgs.clear();
    h.evts.clear();
    h.bbs.clear();
    h.ppool.clear();
    h.gpool.clear();
    hc_package k;
    memset(&k, 0, sizeof(k));
    k.type = type;
    k.num_pulses = n;
    h.pkgs.push_back(k);
    std::vector<int> pc(pulse, pulse + n), gc(gap, gap + n);
    pc.push_back(0); // the entry after the last pulse is part of a package record (zeroed train)
    gc.push_back(0);
    slice_package(h, type, rate, pc.data(), gc.data(), n);
    return (int)h.evts.size();
}

// ---- a native r433b_event_fn that records what r433b_dispatch() hands to decoders ----------
struct Collector {
    std::vector<hc_event> ev;
    std::vector<bitbuffer> bbs;
    int store;
};

void *hc_collector_create(int store)
{
    Collector *c = new Collector();
    c->store = store;
    return c;
}
void hc_collector_destroy(void *c) { delete (Collector *)c; }
void hc_collector_clear(void *c)
{
    ((Collector *)c)->ev.clear();
    ((Collector *)c)->bbs.clear();
}
int hc_collect_cb(void *user, uint32_t package, uint32_t device, struct pulse_data const *pd, struct bitbuffer *bits)
{
    (void)pd;
    Collector *c = (Collector *)user;
    hc_event e;
    e.package = package;
    e.dev = device;
    // the shape a decoder length gate looks at: row count and the longest row (tests of r433b_set_gates)
    unsigned longest = 0;
    for (unsigned r = 0; r < bits->num_rows && r < R433B_BITBUF_ROWS; ++r)
        if (bits->bits_per_row[r] > longest) longest = bits->bits_per_row[r];
    e.ret = (int32_t)(((unsigned)bits->num_rows << 16) | longest);
    e.hash = fnv1a(bits, sizeof(*bits));
    e.bb_idx = 0xffffffffu;
    if (c->store) {
        e.bb_idx = (uint32_t)c->bbs.size();
        c->bbs.push_back(*bits);
    }
    c->ev.push_back(e);
    return 0;
}
size_t hc_collector_count(void *c) { return ((Collector *)c)->ev.size(); }
void const *hc_collector_events(void *c) { return ((Collector *)c)->ev.data(); }
void const *hc_collector_bitbuffers(void *c) { return ((Collector *)c)->bbs.data(); }

size_t hc_num_packages(void *p) { return ((Hc *)p)->pkgs.size(); }
size_t hc_num_events(void *p) { return ((Hc *)p)->evts.size(); }
size_t hc_num_bitbuffers(void *p) { return ((Hc *)p)->bbs.size(); }
size_t hc_num_stage(void *p) { return ((Hc *)p)->am.size(); }
void const *hc_packages(void *p) { return ((Hc *)p)->pkgs.data(); }
void const *hc_events(void *p) { return ((Hc *)p)->evts.data(); }
void const *hc_bitbuffers(void *p) { return ((Hc *)p)->bbs.data(); }
int32_t const *hc_pulse_pool(void *p) { return ((Hc *)p)->ppool.data(); }
int32_t const *hc_gap_pool(void *p) { return ((Hc *)p)->gpool.data(); }
int16_t const *hc_am(void *p) { return ((Hc *)p)->am.data(); }
int16_t const *hc_fm(void *p) { return ((Hc *)p)->fm.data(); }


// the device list k_slice2 walks for one package type (rtl_433_b200/csrc/r433b_host.hpp: slice_list)
int hc_slice_list(void *p, int package_type, uint32_t *out, int cap)
{
    std::vector<unsigned> v = slice_list(((Hc *)p)->devs, package_type);
    for (int i = 0; i < (int)v.size() && i < cap; ++i) out[i] = v[(size_t)i];
    return (int)v.size();
}

// ---- invariants the warp-level kernel code relies on, checked on the product's own functions ----

// k_detect's PULSE fast path: one step of the high-level estimator never lifts it above
// max(high, 64 * (am / 64) + 63), and the "below" threshold never falls when high grows -- so the
// largest sample of a chunk bounds every threshold of the chunk.  Returns the number of violations.
int hc_check_pulse_bound(unsigned seed, int trials)
{
    srand(seed);
    int bad = 0;
    for (int t = 0; t < trials; ++t) {
        // min_level down to -99 dB (min_high 0), min_snr up to 99 dB (ratio * low wraps)
        static float const min_levels[] = {-12.1442f, -13.1442f, -18.1442f, -35.0f, -42.0f, -60.0f, -99.0f};
        static float const min_snrs[] = {9.0f, 1.0f, 60.0f, 99.0f};
        Levels lv = compute_levels(t % 11 == 0, (t % 5 == 0) ? -10.0f : 0.0f, min_levels[t % 7], min_snrs[t / 7 % 4]);
        int const minh = lv.min_high;
        int h = minh + rand() % 30000;
        // AM reaches below zero (to about -350) behind a full-scale sample at a block start, and `low` follows it
        // down; [-2400, 32767] covers the filter's whole reachable range with a margin
        int low = -2401 + rand() % 6400;
        int base = -2400 + rand() % 34400, spread = 1 + rand() % (t % 3 ? 400 : 20000);
        int a[32], top = -512;
        for (int j = 0; j < 32; ++j) {
            int v = base + rand() % spread - spread / 2;
            a[j] = v < -2400 ? -2400 : (v > 32767 ? 32767 : v);
            if (a[j] / 64 > top) top = a[j] / 64; // as k_detect bounds it
        }
        int hmax = 64 * top + 63;
        if (h > hmax) hmax = h;
        Thresholds tmax = det_thresholds(low, hmax, lv);
        for (int j = 0; j < 32; ++j) {
            if (h > hmax) bad++;
            if (det_thresholds(low, h, lv).down > tmax.down) bad++;
            h += a[j] / 64 - (int)((unsigned)h >> 6);
            if (h < minh) h = minh;
        }
        if (h > hmax) bad++;
    }
    return bad;
}

// k_detect's IDLE shortcuts: lowest_up(lmin) is no higher than the trigger level of any `low` >= lmin with `high`
// derived from it, for every Levels -- including those where ratio * low wraps (Levels::monotone == 0).  Levels
// (mode, level_limit, min_level, min_snr) come in `grid` as 4 floats each.  Returns the number of violations, or -1
// when `want_nonmonotone` of the grid points do not have monotone == 0 (the check must reach that branch).
int hc_check_idle_bound(unsigned seed, float const *grid, int n_levels, int trials, int want_nonmonotone)
{
    srand(seed);
    int bad = 0, nonmono = 0;
    for (int g = 0; g < n_levels; ++g) {
        Levels lv = compute_levels((int)grid[4 * g], grid[4 * g + 1], grid[4 * g + 2], grid[4 * g + 3]);
        nonmono += !lv.monotone;
        // exhaustive in `low` near the wrap points and the sign change, random elsewhere
        for (int t = 0; t < trials; ++t) {
            int lmin = t < 4096 ? -2048 + t : -32769 + rand() % 65537;
            int l = lmin + (t & 1 ? rand() % 64 : rand() % 4096);
            if (l > 32768) l = 32768;
            if (lowest_up(lmin, lv) > det_thresholds(l, derived_high(l, lv), lv).up) bad++;
        }
    }
    if (nonmono < want_nonmonotone) return -1;
    return bad;
}

// k_detect's FM on demand: the (provably non-wrapping) low-pass is monotone in its state, so when the
// two ends of the full range have met after some samples, EVERY start state has met them too.
// Runs `trials` random discriminator sequences of `len` samples through the cu8 (cs16 = 0) or cs16
// filter at `rate`; returns -1 on a violation, else how many sequences collapsed.
int hc_check_bracket_rebuild(unsigned seed, int trials, int cs16, unsigned rate, int len, int noise)
{
    srand(seed);
    int a1 = 0, b0 = 0;
    fm_coeffs(cs16, rate, 0.1f, a1, b0);
    long long unity = cs16 ? (1ll << 30) : 16384ll;
    if (!(a1 >= 0 && b0 >= 0 && (long long)a1 + 2ll * b0 <= unity)) return -2;
    int collapsed = 0;
    std::vector<long long> x((size_t)len + 1);
    for (int t = 0; t < trials; ++t) {
        long long lim = cs16 ? 0x7fffffffll : 32767ll;
        long long centre = (long long)(rand() % 2001 - 1000) * (lim / 1000);
        for (int j = 0; j <= len; ++j) {
            long long v = noise ? centre + (long long)(rand() % (2 * noise + 1) - noise) * (cs16 ? 65536 : 1) : centre;
            x[(size_t)j] = v < -lim - 1 ? -lim - 1 : (v > lim ? lim : v);
        }
        auto run = [&](int y) {
            for (int j = 1; j <= len; ++j) {
                long long s = x[(size_t)j] + x[(size_t)j - 1];
                y = cs16 ? iir32(y, a1, b0, s) : iir16_nowrap(y, a1, b0, (int)s);
            }
            return y;
        };
        int lo = run(cs16 ? (int)0x80000000 : -32768), hi = run(cs16 ? 0x7fffffff : 32767);
        if (lo > hi) return -1;
        for (int k = 0; k < 8; ++k) {
            int y0 = cs16 ? (int)((unsigned)rand() * 2654435761u) : rand() % 65536 - 32768;
            int y = run(y0);
            if (y < lo || y > hi) return -1;
        }
        if (lo == hi) collapsed++;
    }
    return collapsed;
}

} // extern "C"
