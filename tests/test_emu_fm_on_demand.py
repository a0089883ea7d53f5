"""CPU: k_detect's single FM path under the SIMT emulator -- the bodies of tests/test_fm_on_demand.py on the kernels'
own source (wrapping filters on cs16 FSK and across time slices, stage arrays and wrapping filters on idle-heavy
streams).  Results must be the oracle's."""
import pytest

import emu
import test_fm_on_demand as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_wrapping_filter_on_cs16_fsk(ctx, devices):
    t.wrapping_filter_on_cs16_fsk(ctx, devices)


def test_emu_wrapping_filter_across_time_slices(ctx, devices):
    t.wrapping_filter_across_time_slices(ctx, devices)


def test_emu_idle_heavy_streams_with_stage_arrays(ctx, devices):
    t.idle_heavy_streams_with_stage_arrays(ctx, devices)


def test_emu_idle_heavy_streams_with_a_wrapping_filter(ctx, devices):
    t.idle_heavy_streams_with_a_wrapping_filter(ctx, devices)
