"""Seeded hostile IQ for the IQ -> package stage (k_front, k_detect): inputs a clipping receiver or a bad capture
produces and that the benchmark's tidy synthetic streams (rtl_433_b200/synth.py) never do.  Each family aims at named
shortcuts of the two kernels and comes with an `evidence` check on the oracle's result (and, where only the kernels
can tell, on the context's timing counters), so that a family which stops reaching its path fails instead of passing.

cs16 inputs stay inside [-32767, 32767]: atan2_int32 on INT32_MIN is a documented divergence (DESIGN.md section 9)."""
import numpy as np

from rtl_433_b200 import synth

RATE = 250000
N = 1 << 18
SMALL_BLOCK = 16384           # samples of a cu8 block of block_bytes = 32768
DEFAULT_BLOCK = 131072        # samples of a cu8 block of the default 262144 bytes
TILE, CHUNK = 2048, 64


class Case:
    """One stream of a family: the IQ, how to read it, and the family's evidence check."""

    def __init__(self, family, seed, iq, fmt=2, rate=RATE, freq=433920000, fpdm=2, levels=None):
        self.family, self.seed, self.iq, self.fmt, self.rate, self.freq, self.fpdm = family, seed, iq, fmt, rate, freq, fpdm
        self.levels = levels or {}

    def __repr__(self):
        return f"{self.family}[seed {self.seed}]"


def _noise(rng, n, sigma=2.0, centre=127.5):
    return rng.standard_normal(2 * n).astype(np.float32) * np.float32(sigma) + np.float32(centre)


def _keyed(x, rng, pos, mask, amp, rate=RATE):
    """Adds a carrier of amplitude `amp` (array or scalar) keyed by `mask` at sample `pos` (float IQ, interleaved)."""
    f = rng.uniform(-60e3, 60e3)
    ph = rng.uniform(0, 2 * np.pi) + 2 * np.pi * f / rate * np.arange(len(mask))
    on = mask.astype(np.float32) * np.float32(1.0) * amp
    x[2 * pos:2 * (pos + len(mask)):2] += on * np.cos(ph).astype(np.float32)
    x[2 * pos + 1:2 * (pos + len(mask)) + 1:2] += on * np.sin(ph).astype(np.float32)


def _cu8(x):
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)


def _train(rng, n_pulses, on, off):
    """On/off mask of n_pulses pulses; on / off are (lo, hi) sample counts, inclusive."""
    seg = []
    for _ in range(n_pulses):
        seg.append(np.ones(int(rng.integers(on[0], on[1] + 1)), np.uint8))
        seg.append(np.zeros(int(rng.integers(off[0], off[1] + 1)), np.uint8))
    return np.concatenate(seg)


# ---------------------------------------------------------------- (255, 255) at block starts ---

SPIKE_OFFSETS = (-1, -1, -1, 0, 1, -2)


def spikes(seed):
    """A tidy OOK capture with single full-scale (255, 255) samples (envelope 32768) just before, at and just after
    block starts of both block sizes: isolated, in pairs, in quiet stretches, in a burst's gap and inside pulses.
    The reference keeps x[-1] as int16 across block calls, so a spike on the last sample of a block enters the next
    one as -32768 and drives its AM below zero for a few dozen samples."""
    rng = np.random.default_rng(1000 + seed)
    iq = synth.ook_stream(seed, n_samples=N, n_bursts=3)
    # a short keyed train across some block starts, so that spikes also land in pulses and gaps
    x = iq.astype(np.float32)
    small_only = [b for b in range(1, N // SMALL_BLOCK) if b * SMALL_BLOCK % DEFAULT_BLOCK]  # default starts stay quiet
    for b in rng.choice(small_only, 3, replace=False):
        start = int(b) * SMALL_BLOCK - int(rng.integers(20, 400))
        m = _train(rng, 30, (8, 60), (8, 60))
        _keyed(x, rng, start, m, np.float32(rng.uniform(40, 100)))
    # the default block start is a quiet stretch even when a burst covers it, so that its spike reaches negative AM
    q = DEFAULT_BLOCK
    x[2 * (q - 300):2 * (q + 100)] = _noise(rng, 400)
    iq = _cu8(x)
    for b in range(1, N // SMALL_BLOCK):
        # always the last sample in front of a default-sized block
        off = -1 if b * SMALL_BLOCK % DEFAULT_BLOCK == 0 else SPIKE_OFFSETS[int(rng.integers(0, len(SPIKE_OFFSETS)))]
        at = b * SMALL_BLOCK + off
        iq[2 * at:2 * at + 2] = 255
        if rng.random() < 0.3 and b * SMALL_BLOCK % DEFAULT_BLOCK:  # a pair (its filter state stays positive)
            iq[2 * (at - 1):2 * at] = 255
    return [Case("spikes", seed, iq)]


def block_start_dips(am, block=SMALL_BLOCK, reach=64):
    """The AM values within `reach` samples behind each block start (the oracle's stage array)."""
    starts = np.arange(block, len(am), block)
    return np.concatenate([am[s:s + reach] for s in starts]) if len(starts) else np.zeros(0, np.int16)


def spikes_evidence(case, ref, block):
    am = ref["am"]
    assert block_start_dips(am, block).min() < 0, f"{case}: no negative AM next to a block start"


# ---------------------------------------------------------------- full scale ---

def rails(seed):
    """Long full-scale stretches, saturated OOK bursts and alternating rails: AM up to the top of int16, where
    iir16_nowrap, the chunk and tile bounds and the thresholds' int16 casts live."""
    rng = np.random.default_rng(2000 + seed)
    x = _noise(rng, N)
    pos = 3000
    while pos < N - 30000:
        kind = int(rng.integers(0, 3))
        if kind == 0:    # a saturated carrier: both rails reached every cycle
            m = _train(rng, int(rng.integers(5, 40)), (20, 400), (20, 400))
            _keyed(x, rng, pos, m, np.float32(400.0))
        elif kind == 1:  # a constant full-scale stretch at a corner of the IQ square
            ln = int(rng.integers(300, 6000))
            x[2 * pos:2 * (pos + ln)] = [(0, 0), (255, 255), (255, 0), (0, 255)][int(rng.integers(0, 4))] * ln
            m = np.ones(ln, np.uint8)
        else:            # alternating rails sample by sample
            ln = int(rng.integers(300, 6000))
            alt = np.where(np.arange(ln) % 2 == 0, 0.0, 255.0).astype(np.float32)
            x[2 * pos:2 * (pos + ln):2] = alt
            x[2 * pos + 1:2 * (pos + ln) + 1:2] = alt[::-1]
            m = np.ones(ln, np.uint8)
        pos += len(m) + int(rng.integers(3000, 12000))
    return [Case("rails", seed, _cu8(x))]


def rails_evidence(case, ref, block):
    assert ref["am"].max() > 32000, f"{case}: AM never came near the top of int16"


# ---------------------------------------------------------------- glitches ---

def glitches(seed):
    """Trains of 1-12-sample pulses and gaps mixed into regular pulse trains, at levels around the thresholds:
    spurious pulses and gaps mid-package, burst_run's ballot scans, the hysteresis band."""
    rng = np.random.default_rng(3000 + seed)
    x = _noise(rng, N)
    pos = 2500
    while pos < N - 20000:
        parts = []
        for _ in range(int(rng.integers(3, 12))):
            if rng.random() < 0.5:
                parts.append(_train(rng, int(rng.integers(2, 20)), (10, 80), (10, 120)))  # regular pulses
            else:
                parts.append(_train(rng, int(rng.integers(1, 30)), (1, 12), (1, 12)))    # glitches
        m = np.concatenate(parts)
        amp = np.where(m > 0, np.float32(rng.uniform(18, 90)), 0).astype(np.float32)
        amp *= np.float32(1.0) + rng.uniform(-0.15, 0.15, len(m)).astype(np.float32)  # levels around the thresholds
        _keyed(x, rng, pos, np.ones(len(m), np.uint8), amp)
        pos += len(m) + int(rng.integers(2000, 9000))
    return [Case("glitches", seed, _cu8(x))]


def ended_by_spurious(pkg, rate):
    """An OOK package of fewer than 1200 pulses whose last gap is shorter than every gap limit: a spurious pulse ended
    it (src/pulse_detect.c:341-350; the limits need a gap over 10 ms)."""
    n = pkg["num_pulses"]
    return pkg["type"] == 1 and 0 < n < 1200 and pkg["end_ago"] != 0 and int(pkg["gap"][n - 1]) <= 10 * (rate // 1000)


def glitches_evidence(case, ref, block):
    assert any(ended_by_spurious(p, case.rate) for p in ref["packages"]), f"{case}: no package ended by a spurious pulse"


# ---------------------------------------------------------------- drifting floors ---

def floors(seed):
    """A noise floor that ramps slowly, steps, carries a DC offset, and a tone whose amplitude hugs the trigger level,
    between real bursts: idle_skip's brackets and condition on the tracker, derived_high, lead_in."""
    rng = np.random.default_rng(4000 + seed)
    t = np.arange(N, dtype=np.float32)
    sigma = np.float32(1.0) + np.float32(rng.uniform(1, 6)) * (np.float32(0.5) + np.float32(0.5) * np.sin(t * np.float32(2 * np.pi / rng.uniform(4e4, 2e5))))
    step = np.where(t > rng.uniform(0.3, 0.7) * N, np.float32(rng.uniform(1, 4)), np.float32(1.0))
    x = rng.standard_normal(2 * N).astype(np.float32) * np.repeat(sigma * step, 2)
    dc = rng.uniform(-12, 12, 2).astype(np.float32)
    x[0::2] += np.float32(127.5) + dc[0]
    x[1::2] += np.float32(127.5) + dc[1]
    # a tone hugging the level at which the detector would trigger, slowly wandering around it
    tlen = int(rng.integers(20000, 60000))
    tpos = int(rng.integers(10000, N - tlen - 10000))
    hug = np.float32(rng.uniform(6, 16)) * (np.float32(1.0) + np.float32(0.3) * np.sin(np.arange(tlen, dtype=np.float32) * np.float32(rng.uniform(1e-4, 1e-3))))
    _keyed(x, rng, tpos, np.ones(tlen, np.uint8), hug)
    for _ in range(3):  # real bursts: packages to find after the floor has moved
        m = _train(rng, int(rng.integers(20, 60)), (60, 200), (60, 200))
        p = int(rng.integers(5000, N - len(m) - 5000))
        _keyed(x, rng, p, m, np.float32(rng.uniform(50, 100)))
    return [Case("floors", seed, _cu8(x))]


def floors_evidence(case, ref, block, timing=None):
    assert ref["packages"], f"{case}: no packages"
    if timing is not None:
        assert timing["idle_skipped"] > 0, f"{case}: no tile skipped: {timing}"


# ---------------------------------------------------------------- exact plateaus ---

def plateaus(seed):
    """Exactly constant IQ at random levels with abrupt steps on tile, chunk and block positions (and off them), and
    short bursts between: the AM filter sits on one of several fixed points of its floor map, so k_front's guesses
    land on the wrong one and have to be redone or repaired; the walk's brackets cannot collapse."""
    rng = np.random.default_rng(5000 + seed)
    x = np.zeros(2 * N, np.float32)
    pos = 0
    while pos < N:
        grid = (CHUNK, TILE, SMALL_BLOCK, 1)[int(rng.integers(0, 4))]
        ln = max(grid, int(rng.integers(1, 12)) * grid) if grid > 1 else int(rng.integers(50, 5000))
        ln = min(ln, N - pos)
        x[2 * pos:2 * (pos + ln)] = np.tile(rng.integers(60, 200, 2).astype(np.float32), ln)
        pos += ln
    for _ in range(4):
        m = _train(rng, int(rng.integers(10, 40)), (40, 200), (40, 200))
        p = int(rng.integers(1000, N - len(m) - 1000))
        x[2 * p:2 * (p + len(m))] = 127.0
        _keyed(x, rng, p, m, np.float32(rng.uniform(60, 110)))
    return [Case("plateaus", seed, _cu8(x))]


def plateaus_evidence(case, ref, block, timing=None):
    if timing is not None:
        assert timing["front_repairs"] > 0 or timing["front_redone"] > 0, f"{case}: no guess redone or repaired: {timing}"


# ---------------------------------------------------------------- tile phases ---

PHASES = (0, 1, 63, 64, 2047)


def tile_phases(seed):
    """A pulse train whose first pulse starts on sample 0, 1, 63, 64 or 2047 of a tile, or on the last sample of a
    block, behind a quiet stretch: the tile hand-over and the walk's phases at tile ends."""
    out = []
    for k, ph in enumerate(PHASES + (-1,)):
        rng = np.random.default_rng(6000 + 10 * seed + k)
        x = _noise(rng, N)
        start = (40 + 3 * k + 5 * seed) * TILE + ph if ph >= 0 else (2 + seed % 5) * SMALL_BLOCK - 1
        m = _train(rng, int(rng.integers(15, 40)), (30, 150), (30, 150))
        _keyed(x, rng, start, m, np.float32(rng.uniform(60, 110)))
        c = Case("tile_phases", seed, _cu8(x))
        c.start = start
        out.append(c)
    return out


def tile_phases_evidence(case, ref, block):
    offs = [p["offset"] for p in ref["packages"] if p["type"] == 1]
    assert offs and min(abs(int(o) - case.start) for o in offs) <= 2, f"{case}: no package at sample {case.start}: {offs}"


# ---------------------------------------------------------------- 1200-pulse trains ---

def long_trains(seed):
    """Trains of more than 1200 pulses of 10-12 samples: PD_MAX_PULSES reached in burst_run's GAP scan or in
    det_step, at every phase against the tile grid."""
    rng = np.random.default_rng(7000 + seed)
    x = _noise(rng, N)
    m = _train(rng, 1250 + int(rng.integers(0, 100)), (10, 12), (24, 48))  # gaps the filter cannot close
    _keyed(x, rng, int(rng.integers(2000, 9000)), m, np.float32(rng.uniform(50, 110)))
    return [Case("long_trains", seed, _cu8(x))]


def long_trains_evidence(case, ref, block):
    assert any(p["type"] == 1 and p["num_pulses"] == 1200 for p in ref["packages"]), f"{case}: no 1200-pulse package"


# ---------------------------------------------------------------- cs16 FSK at every amplitude ---

FSK_RATE = 1024000


def fsk_cs16(seed):
    """cs16 with rail values +-32767 and large DC offsets, and 2-FSK bursts from a few LSB up to the rails:
    mag_cs16, atan32, first_run's FSK sub-detector and the FM windows; both FSK pulse detectors."""
    rng = np.random.default_rng(8000 + seed)
    n = N
    dc = rng.uniform(-3000, 3000, 2)
    x = rng.standard_normal(2 * n) * rng.uniform(2, 60)
    x[0::2] += dc[0]
    x[1::2] += dc[1]
    pos = 5000
    # one burst that stands well above the DC offset, then a few LSB .. well past the rails
    for amp in [rng.uniform(4000, 14000) + 2 * np.abs(dc).max()] + list(rng.uniform(0, 1, 4) ** 3 * 45000 + 6):
        bits = np.concatenate([np.tile([1, 0], 16), rng.integers(0, 2, 96)])
        spb = rng.uniform(60, 140) * FSK_RATE / 1e6
        blen = int(np.ceil(len(bits) * spb))
        if pos + blen + 8000 > n:
            break
        idx = np.minimum((np.arange(blen) / spb).astype(np.int64), len(bits) - 1)
        dev = rng.uniform(15e3, 60e3)
        freq = np.where(bits[idx] > 0, dev, -dev) + rng.uniform(-10e3, 10e3)
        ph = rng.uniform(0, 2 * np.pi) + 2 * np.pi * np.cumsum(freq) / FSK_RATE
        x[2 * pos:2 * (pos + blen):2] += amp * np.cos(ph)
        x[2 * pos + 1:2 * (pos + blen) + 1:2] += amp * np.sin(ph)
        pos += blen + int(rng.integers(6000, 20000))
    iq = np.clip(np.rint(x), -32767, 32767).astype(np.int16)
    return [Case("fsk_cs16", seed, iq, fmt=4, rate=FSK_RATE, freq=868000000, fpdm=fpdm) for fpdm in (2, 0)]


def fsk_cs16_evidence(case, ref, block):
    if case.fpdm == 0:  # the classic detector misses some of these bursts: compared, but not required to find one
        return
    assert any(p["type"] == 2 for p in ref["packages"]), f"{case}: no FSK package"


FAMILIES = {
    "spikes": (spikes, spikes_evidence),
    "rails": (rails, rails_evidence),
    "glitches": (glitches, glitches_evidence),
    "floors": (floors, floors_evidence),
    "plateaus": (plateaus, plateaus_evidence),
    "tile_phases": (tile_phases, tile_phases_evidence),
    "long_trains": (long_trains, long_trains_evidence),
    "fsk_cs16": (fsk_cs16, fsk_cs16_evidence),
}
TIMED = {"floors", "plateaus"}  # evidence that only the kernels' counters can give
