"""CPU: k_detect's idle-tile skip under the SIMT emulator -- the bodies of tests/test_idle_skip.py on the kernels' own
source, and once more with R4_FORCE_REWALK=1, which makes every skipped run fail its resolution so that the
backstop walks it again from the exact state in front of it.  Results must not change either way."""
import os
import subprocess

import pytest

import emu
import test_idle_skip as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

REWALK_SO = os.path.join(emu.HERE, "_build", "libr433b_emu_rewalk.so")


def build_rewalk():
    """emu.build()'s library with every skipped run walked again, beside the regular emulated build."""
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    os.makedirs(os.path.dirname(REWALK_SO), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR4_FORCE_REWALK=1", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", REWALK_SO])
    return REWALK_SO


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_idle_heavy_streams(ctx, devices):
    t.idle_heavy_streams_match_the_oracle_and_the_reference(ctx, devices)


def test_emu_bursts_right_behind_a_skipped_run(ctx, devices):
    t.bursts_right_behind_a_skipped_run(ctx, devices)


def test_emu_ragged_lengths_and_small_blocks_with_skipping(ctx, devices):
    t.ragged_lengths_and_small_blocks_with_skipping(ctx, devices)


def test_emu_time_slices_with_skipping(ctx, devices):
    t.time_slices_with_skipping(ctx, devices)


def test_emu_repairs_between_skipped_runs(devices, monkeypatch):
    t.repairs_between_skipped_runs(devices, monkeypatch)


def test_emu_every_skipped_run_walked_again(devices):
    """R4_FORCE_REWALK=1: the backstop takes every run, so nothing counts as skipped and results stay exact."""
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = build_rewalk(), None
    try:
        c = lib.Context(0)
        c.set_devices(devices)
        try:
            streams = t.idle_heavy()
            got, tm = t.run_skipping(c, streams)
            o = t.oracle_for(devices, stages=False)
            for i, s in enumerate(streams):
                t.check(got[i], o.run(s, 2), f"re-walked stream {i}")
            assert tm["idle_rewalks"] > 0 and tm["idle_skipped"] == 0, tm
            got, tm = t.run_skipping(c, streams, block_bytes=32768)
            for i, s in enumerate(streams):
                t.check(got[i], o.run(s, 2, block_bytes=32768), f"re-walked stream {i}, small blocks")
            assert tm["idle_rewalks"] > 0, tm
        finally:
            c.close()
    finally:
        lib.LIB_PATH, lib._lib = old
