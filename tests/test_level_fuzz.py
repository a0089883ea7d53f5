"""-m gpu: the hostile-IQ fuzz (tests/test_front_fuzz.py) across the detector's level settings (`-Y ampest|magest`,
`-Y level=`, `-Y minlevel=`, `-Y minsnr=`, r433b_set_levels).  k_detect's shortcuts each rest on a property of the
thresholds those settings make -- the trigger level growing with `low`, `high` never below zero, negative AM below
`down` -- so every family runs at every point of GRID against the oracle with nothing relaxed: packages, widths,
every event and both stage arrays, with and without stage arrays, at both block sizes, on every seed.  The regimes
that once parted from the reference also run through the pipelined host path and chained batches, and against the
compiled reference where it is present.  tests/test_oracle_vs_ref.py pins the oracle to the reference on the same
grid; tests/test_emu_level_fuzz.py runs these bodies under the SIMT emulator."""
import ctypes as C

import pytest

import helpers
import hostile_iq as H
import test_front_fuzz as t
from oracle import orc
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

DEFAULT = dict(use_mag_est=0, level_limit=0.0, min_level=-12.1442, min_snr=9.0)

# one setting at a time from the defaults, in envelope (0) and magnitude (1) mode
AXES = {
    "level_limit": (0.0, -1.0, -8.0, -20.0, -30.0, -40.0, -60.0),
    "min_level": (-1.0, -3.0, -12.1442, -25.0, -35.0, -40.0, -42.0, -60.0, -99.0),  # min_high reaches 1, then 0
    "min_snr": (1.0, 3.0, 9.0, 20.0, 46.0, 50.0, 60.0, 99.0),  # ratio * 32767 crosses 2^31 at 48.2 dB (envelope)
}
COMBINED = (
    dict(use_mag_est=1, min_level=-80.0, min_snr=60.0),
    dict(use_mag_est=0, level_limit=-30.0, min_level=-60.0),
    dict(use_mag_est=0, min_level=-40.0, min_snr=1.0),
)
GRID = [dict(use_mag_est=m, **{k: v}) for m in (0, 1) for k, vs in AXES.items() for v in vs] + list(COMBINED)

# The regimes that parted from the reference, one setting each (the pipelined / chained runs take these)
REGIMES = (dict(level_limit=-30.0), dict(min_level=-40.0), dict(min_level=-99.0), dict(min_snr=60.0),
           dict(use_mag_est=1, level_limit=-40.0))

# Reproductions: (family, levels) on seed 0 at the default block size, each of which the kernels once got wrong.
#  - a low fixed level or a long first pulse: first_run fed the classic FSK sub-detector up to 32 samples per trip
#    while it reads the FSK train back (short pulses merged), so a lane could read an entry a faster lane had already
#    overwritten for a later sample, and the last lane's train won;
#  - a fixed level of 1 (envelope, -40 dB): the first pulse's GAP_START fed the FSK sub-detector its 17th pulse on
#    the sample it moved to GAP, and burst_run, which leaves the FSK hand-over out, walked past the next GAP_START;
#  - min_snr = 60 dB: ratio * low wraps above low = 2147, derived_high() is no longer monotone and the IDLE
#    shortcuts' trigger bound at the lowest reachable `low` was not the lowest trigger level.
REPRODUCTIONS = {
    "fixed_level_30_floors": ("floors", dict(level_limit=-30.0)),
    "magnitude_fixed_level_40_glitches": ("glitches", dict(use_mag_est=1, level_limit=-40.0)),
    "magnitude_fixed_level_40_floors": ("floors", dict(use_mag_est=1, level_limit=-40.0)),
    "magnitude_fixed_level_40_rails": ("rails", dict(use_mag_est=1, level_limit=-40.0)),
    "min_level_40_spikes": ("spikes", dict(min_level=-40.0)),
    "min_level_60_glitches": ("glitches", dict(min_level=-60.0)),
    "min_level_99_glitches": ("glitches", dict(min_level=-99.0)),
    "min_snr_60_glitches": ("glitches", dict(min_snr=60.0)),
    "fixed_level_40_tile_phases": ("tile_phases", dict(level_limit=-40.0)),
}


def tag(levels):
    return ",".join(f"{k}={v:g}" for k, v in levels.items())


def detector_levels(levels):
    """(fixed_high, min_high, ratio, max_high) as the oracle derives them (src/pulse_detect.c:86-98)."""
    lv = dict(DEFAULT, **levels)
    out = (C.c_int32 * 4)()
    orc.lib().orc_detector_levels(int(lv["use_mag_est"]), lv["level_limit"], lv["min_level"], lv["min_snr"], out)
    return tuple(out)


def equals_default(levels):
    """Points whose derived levels are the defaults' (envelope mode: level_limit 0 or -60, whose fixed level
    truncates to 0, i.e. adaptive; and the default values themselves)."""
    return detector_levels(levels) == detector_levels({})


def same_result(a, b):
    return not helpers.compare_results(a, b, "", stages=True)


_baselines = {}


def baseline(devices, name, seeds, blocks):
    """The oracle's results at the default levels (made once per process), keyed like run_family's collect list."""
    key = (name, tuple(seeds), tuple(blocks))
    if key not in _baselines:
        _baselines[key] = t.oracle_results(devices, [c for s in seeds for c in t.family_cases(name, s)], blocks)
    return _baselines[key]


def level_point(ctx, devices, levels, seeds, blocks=t.BLOCKS, names=tuple(H.FAMILIES)):
    """Every family in `names` at `levels` against the oracle.  The point must not be inert: on at least one family
    the oracle's result differs from its result at the default levels -- except where the derived levels are the
    defaults', where every result must be the default one."""
    moved = False
    for name in names:
        got = []
        t.run_family(ctx, devices, name, seeds, blocks=blocks, levels=levels, evidence=False, collect=got)
        if moved and not equals_default(levels):
            continue
        base = baseline(devices, name, seeds, blocks)
        same = [same_result(base[(id(c), bb)], want) for c, bb, want in got]
        if equals_default(levels):
            assert all(same), f"{tag(levels)} derives the default levels but {name} differs from the default"
        moved = moved or not all(same)
    assert moved or equals_default(levels), f"{tag(levels)}: inert on every family"


def test_grid_shape():
    """The grid reaches the edges it is meant to: a fixed level that truncates to 0 (adaptive), min_high 1 and 0,
    and ratio * 32767 past 2^31 in envelope mode only from 49 dB on and in magnitude mode only above 96 dB."""
    assert detector_levels(dict(level_limit=-60.0))[0] == 0
    assert detector_levels(dict(use_mag_est=1, level_limit=-60.0))[0] > 0
    assert {detector_levels(g)[1] for g in GRID} >= {0, 1}
    for mode, first_wrap in ((0, 50.0), (1, 99.0)):
        for snr in AXES["min_snr"]:
            ratio = detector_levels(dict(use_mag_est=mode, min_snr=snr))[2]
            assert (abs(ratio * 32767) >= 2 ** 31) == (snr >= first_wrap), (mode, snr, ratio)
    # 99 dB in envelope mode: 7.9e9 does not fit an int; the conversion gives INT_MIN, as in the reference on x86
    assert detector_levels(dict(min_snr=99.0))[2] == -2 ** 31
    assert sum(equals_default(g) for g in GRID) == 4  # envelope: level_limit 0 and -60, min_level, min_snr defaults


@pytest.mark.gpu
@pytest.mark.parametrize("levels", GRID, ids=[f"{'mag' if g['use_mag_est'] else 'env'}:{tag(g)}" for g in GRID])
def test_level_grid(ctx, devices, levels):
    level_point(ctx, devices, levels, t.SEEDS)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REPRODUCTIONS))
def test_reproduction(ctx, devices, name):
    family, levels = REPRODUCTIONS[name]
    t.run_family(ctx, devices, family, [0], blocks=(0,), levels=levels, evidence=False)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", REGIMES, ids=[tag(g) for g in REGIMES])
def test_pipelined_and_chained_levels(ctx, devices, levels):
    t.pipelined_and_chained(ctx, devices, t.SEEDS[:3], levels=levels)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", REGIMES, ids=[tag(g) for g in REGIMES])
def test_against_reference_levels(ctx, devices, levels):
    for name in H.FAMILIES:
        t.against_reference(ctx, list(t.family_cases(name, 0)), levels=levels)
