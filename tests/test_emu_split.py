"""CPU: segmented replay under the SIMT emulator (tests/emu.py) -- the bodies of tests/test_split.py at smaller sizes, on
the kernels' own source: the seed comparison, the gather / scatter of the rewalks and the merge, including every seed
rejected and one arena overflow under the exact-allocation build."""
import os
import subprocess

import pytest

import emu
import test_split as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_ook_bursts(ctx, devices):
    t.ook_bursts(ctx, devices, n=1 << 16)


def test_emu_burst_over_many_segments(ctx, devices):
    t.burst_over_many_segments(ctx, devices, n_pulses=150)


def test_emu_open_packages_at_segment_starts(ctx, devices, monkeypatch):
    t.open_packages_at_segment_starts(ctx, devices, monkeypatch)


def test_emu_fsk_fm_on(ctx, devices):
    t.fsk_fm_on(ctx, devices, n=1 << 16)


def test_emu_cs8_and_cf32(ctx, devices):
    t.cs8_and_cf32(ctx, devices, n=1 << 16)


def test_emu_levels_and_low_pass(ctx, devices):
    t.levels_and_low_pass(ctx, devices, n=1 << 16)


def test_emu_ragged_mixed_batch(ctx, devices):
    t.ragged_mixed_batch(ctx, devices, n=1 << 16)


def test_emu_segment_sizes(ctx, devices):
    t.segment_sizes(ctx, devices, n=1 << 16)


def test_emu_spoiled_seeds(devices, monkeypatch):
    t.spoiled_seeds(devices, monkeypatch, n=1 << 16)


def test_emu_unsplit_schedules(ctx, devices):
    t.unsplit_schedules(ctx, devices)


def test_emu_arena_overflow_exact_alloc(devices, monkeypatch):
    """The overflow rerun with every buffer ending at its cap (-DR433B_EXACT_ALLOC)."""
    so = os.path.join(emu.HERE, "_build", "libr433b_emu_split_exact.so")
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR433B_EXACT_ALLOC", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", so])
    monkeypatch.setenv("SIMT_GUARD", "back")  # read by the library's first allocation
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = so, None
    try:
        t.arena_overflow(devices, monkeypatch, n=1 << 16)
    finally:
        lib.LIB_PATH, lib._lib = old
