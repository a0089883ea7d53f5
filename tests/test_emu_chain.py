"""CPU: chained batches under the SIMT emulator (tests/emu.py) -- the bodies of tests/test_chain.py on the kernels' own
source, where every IQ and AM index is also asserted not to go below the chunk start."""
import pytest

import emu
import test_chain as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_ook_cu8_every_and_random_boundaries(ctx, devices):
    t.ook_cu8_every_and_random_boundaries(ctx, devices)


def test_emu_fsk_cs16_cut_in_first_pulses(ctx, devices):
    t.fsk_cs16_cut_in_first_pulses(ctx, devices)


def test_emu_long_ook_package_folded_at_boundaries(ctx, devices):
    t.long_ook_package_folded_at_boundaries(ctx, devices)


def test_emu_spoiled_first_tiles(devices, monkeypatch):
    t.spoiled_first_tiles(devices, monkeypatch)


def test_emu_cs8_and_cf32(ctx, devices):
    t.cs8_and_cf32(ctx, devices)


def test_emu_ragged_slots(ctx, devices):
    t.ragged_slots(ctx, devices)


def test_emu_time_sliced_chains(ctx, devices):
    t.time_sliced_chains(ctx, devices)


def test_emu_errors(ctx, devices):
    t.errors(ctx, devices)


def test_emu_decoders_and_analyzer(devices):
    t.decoders_and_analyzer(devices)


def test_emu_command_line_chunks(capsys, tmp_path):
    t.command_line_chunks(capsys, tmp_path)
