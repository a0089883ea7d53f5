"""CPU: the signal grabber on chained batches under the SIMT emulator (tests/emu.py) -- k_grab_ring and k_grab's ring
segments on the kernels' own source, with the bodies of tests/test_chain_grab.py: every slot's chained grabs against
one unchained batch of its files, once with the lanes of every warp in descending order."""
import os
import subprocess
import sys

import pytest

import emu
import test_chain_grab as t
import test_grab as tg
from rtl_433_b200 import lib


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


@pytest.fixture(scope="module")
def devices():
    return lib.default_device_table()


@pytest.fixture(scope="module")
def ctx(devices):
    c = lib.Context(0)
    c.set_devices(devices)
    yield c
    c.close()


def test_emu_cadences_slots_and_files(ctx):
    t.cadences_slots_and_files(ctx)


def test_emu_cs8(ctx):
    t.cadences_slots_and_files(ctx, fmt=lib.FMT_CS8)


def test_emu_chunks_larger_than_the_ring(ctx):
    t.chunks_larger_than_the_ring(ctx)


@pytest.mark.parametrize("fmt", [lib.FMT_CU8, lib.FMT_CS16], ids=["cu8", "cs16"])
def test_emu_unaligned_ring_positions(ctx, fmt):
    t.unaligned_ring_positions(ctx, fmt)


def test_emu_cs16_and_cf32(ctx):
    t.fsk_formats(ctx)


def test_emu_arena_overflow_rerun(devices, monkeypatch):
    t.arena_overflow_rerun(devices, monkeypatch)


@tg.needs_ref
def test_emu_mode_known_with_reference_decoders():
    decoders = tg.Decoders()
    c = lib.Context(0)
    try:
        c.set_devices(decoders.devices)
        t.cadences_slots_and_files(c, lib.GRAB_KNOWN, decoders)
    finally:
        c.close()
        decoders.close()


def test_emu_state_errors(devices):
    t.state_errors(devices)


def test_emu_reverse_lanes():
    """Lanes in descending order (SIMT_REVERSE=1): the shuffled words of k_grab_ring (appends from unaligned ring
    positions, cs8 flipped on the way) and of k_grab."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import emu; emu.use()\n"
            "import test_chain_grab as t\n"
            "from rtl_433_b200 import lib\n"
            "c = lib.Context(0); c.set_devices(lib.default_device_table())\n"
            "t.unaligned_ring_positions(c, lib.FMT_CS8)\n"
            "c.close()\n") % (here, os.path.dirname(here))
    assert subprocess.call([sys.executable, "-c", code], env=dict(os.environ, SIMT_REVERSE="1")) == 0
