"""CPU: the hostile-IQ fuzz of tests/test_front_fuzz.py under the SIMT emulator, on the kernels' own source, with
fewer seeds: once on the regular emulated build, once with R4_FORCE_REWALK=1 (every skipped idle run walked again
from the exact state in front of it) and once with the lanes scheduled in descending order."""
import os
import subprocess
import sys

import pytest

import emu
import hostile_iq as H
import test_front_fuzz as t
from rtl_433_b200 import lib
from test_emu_idle_skip import build_rewalk
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

SEEDS = range(2)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


@pytest.mark.parametrize("name", list(H.FAMILIES))
def test_emu_family(ctx, devices, name):
    t.run_family(ctx, devices, name, SEEDS)


def test_emu_levels(ctx, devices):
    t.levels(ctx, devices, SEEDS[:1])


def test_emu_pipelined_and_chained(ctx, devices):
    t.pipelined_and_chained(ctx, devices, SEEDS[:1])


def test_emu_every_skipped_run_walked_again(devices):
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = build_rewalk(), None
    try:
        c = lib.Context(0)
        c.set_devices(devices)
        try:
            for name in H.FAMILIES:
                # this build counts nothing as skipped: the floors family shows its rewalks instead
                t.run_family(c, devices, name, SEEDS[:1], evidence=name != "floors")
                if name == "floors":
                    assert c.timing()["idle_rewalks"] > 0, c.timing()
        finally:
            c.close()
    finally:
        lib.LIB_PATH, lib._lib = old


def test_emu_reverse_schedule():
    """Lanes in descending order (SIMT_REVERSE=1) on one seed of every family."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys;sys.path[:0]=[%r,%r];import emu;emu.use();import hostile_iq as H,test_front_fuzz as t;"
            "from rtl_433_b200 import lib;devs=lib.default_device_table();c=lib.Context(0);c.set_devices(devs)\n"
            "for n in H.FAMILIES: t.run_family(c,devs,n,[5])\n") % (here, emu.ROOT)
    assert subprocess.call([sys.executable, "-c", code], env=dict(os.environ, SIMT_REVERSE="1")) == 0
