"""CPU checks (on the product's own __host__ __device__ functions, through tests/host_core.cpp) of
the two invariants the warp-level shortcuts of k_detect rest on; the shortcuts themselves are
covered bit-for-bit by the -m gpu parity tests."""
import ctypes as C

import numpy as np

import helpers
from rtl_433_b200 import lib


def _lib():
    L = C.CDLL(helpers.build_hostcore())
    L.hc_check_pulse_bound.argtypes = [C.c_uint, C.c_int]
    L.hc_check_bracket_rebuild.argtypes = [C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_int]
    return L


def test_pulse_threshold_bound():
    """PULSE fast path: the chunk maximum bounds the high estimate and every "below" threshold."""
    assert _lib().hc_check_pulse_bound(1, 200000) == 0


def test_idle_trigger_bound_on_the_level_grid():
    """IDLE shortcuts: lowest_up(lmin) never lies above the trigger level of a `low` >= lmin, at every level of the
    level fuzz's grid -- among them the min_snr settings where ratio * low wraps and derived_high() is not monotone."""
    import test_level_fuzz as lf
    grid = [dict(lf.DEFAULT, **g) for g in lf.GRID]
    flat = np.array([[g["use_mag_est"], g["level_limit"], g["min_level"], g["min_snr"]] for g in grid], np.float32)
    L = _lib()
    L.hc_check_idle_bound.argtypes = [C.c_uint, C.c_void_p, C.c_int, C.c_int, C.c_int]
    # not monotone: envelope mode at 50 and 60 dB, magnitude mode at 99 dB (envelope mode at 99 dB has ratio INT_MIN,
    # which makes every ratio * low 0 or INT_MIN: `high` is min_high throughout)
    assert L.hc_check_idle_bound(3, flat.ctypes.data, len(grid), 20000, 3) == 0


def test_fm_filter_state_rebuild_is_sound_and_usually_converges():
    """FM on demand: monotone filter => once the two extreme start states meet, all states have met.
    A live (noisy) discriminator makes them meet within one 1024/512-sample tile; an exactly
    constant one does not -- the case the kernel handles by walking forward from the last exact state."""
    L = _lib()
    for cs16, rate, tile in ((0, 250000, 1024), (0, 1024000, 1024), (1, 1024000, 512), (1, 250000, 512)):
        n = L.hc_check_bracket_rebuild(7, 400, cs16, rate, tile, 300)
        assert n >= 0, "a start state escaped the bracket"
        assert n >= 396, f"only {n}/400 noisy sequences converged within one tile (cs16={cs16}, rate={rate})"
        n = L.hc_check_bracket_rebuild(7, 50, cs16, rate, tile, 0)
        assert n >= 0
    # constant input: the floor map keeps distinct fixed points apart for at least some levels
    assert L.hc_check_bracket_rebuild(9, 200, 0, 250000, 1024, 0) < 200


def test_slice_work_lists_cover_every_device_once_in_slicer_order():
    """k_slice2 takes these lists device by device: every device that takes the package type appears
    exactly once and nothing else does; devices of one modulation stay together, modulations ascend,
    and within a modulation the order is (reset_limit, short_width), then registration."""
    devs = lib.default_device_table(include_disabled=True)
    hc = helpers.HostCore()
    hc.add_devices(devs)
    hc.L.hc_slice_list.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    for ptype, takes in ((1, lambda m: 3 <= m <= 13 and m != 7), (2, lambda m: 16 <= m <= 18)):
        buf = np.zeros(4096, np.uint32)
        n = hc.L.hc_slice_list(hc.h, ptype, buf.ctypes.data, len(buf))
        lst = [int(x) for x in buf[:n]]
        want = [i for i, d in enumerate(devs) if takes(d["modulation"])]
        assert sorted(lst) == want
        # the device table holds floats (r433b_device): compare in float32 as slice_list does
        key = [(devs[i]["modulation"], np.float32(devs[i]["reset_limit"]), np.float32(devs[i]["short_width"]), i) for i in lst]
        assert key == sorted(key), "modulations contiguous and ascending, then (reset_limit, short_width)"
