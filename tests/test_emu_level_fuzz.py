"""CPU: the level fuzz of tests/test_level_fuzz.py under the SIMT emulator, on the kernels' own source, on seed 0:
every reproduction, one point of each level axis on every family, the pipelined host path and chained batches at
min_snr = 60 dB, and the reproductions once more with the lanes scheduled in descending order."""
import os
import subprocess
import sys

import pytest

import emu
import test_front_fuzz as t
import test_level_fuzz as lf
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

AXIS_POINTS = (dict(use_mag_est=1, level_limit=-40.0), dict(min_level=-42.0), dict(min_snr=50.0))


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


@pytest.mark.parametrize("name", list(lf.REPRODUCTIONS))
def test_emu_reproduction(ctx, devices, name):
    family, levels = lf.REPRODUCTIONS[name]
    t.run_family(ctx, devices, family, [0], blocks=(0,), levels=levels, evidence=False)


@pytest.mark.parametrize("levels", AXIS_POINTS, ids=[lf.tag(g) for g in AXIS_POINTS])
def test_emu_level_point(ctx, devices, levels):
    lf.level_point(ctx, devices, levels, [0], blocks=(0,))


def test_emu_pipelined_and_chained_levels(ctx, devices):
    t.pipelined_and_chained(ctx, devices, [0], levels=dict(min_snr=60.0))


def test_emu_reverse_schedule():
    """Lanes in descending order (SIMT_REVERSE=1) on every reproduction."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys;sys.path[:0]=[%r,%r];import emu;emu.use();import test_front_fuzz as t,test_level_fuzz as lf;"
            "from rtl_433_b200 import lib;devs=lib.default_device_table();c=lib.Context(0);c.set_devices(devs)\n"
            "for f, lv in lf.REPRODUCTIONS.values(): t.run_family(c,devs,f,[0],blocks=(0,),levels=lv,evidence=False)\n"
            ) % (here, emu.ROOT)
    assert subprocess.call([sys.executable, "-c", code], env=dict(os.environ, SIMT_REVERSE="1")) == 0
