"""CPU: segmented replay on chained batches under the SIMT emulator (tests/emu.py) -- the bodies of
tests/test_chain_split.py at smaller sizes, on the kernels' own source: the chain's state into a chunk's first segment
and out of its last, the seq carried through the merge, and one arena overflow under the exact-allocation build."""
import os
import subprocess

import pytest

import emu
import test_chain_split as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_ook_bursts_across_boundaries(ctx, devices):
    t.ook_bursts_across_boundaries(ctx, devices, n=1 << 17)


def test_emu_fsk_minmax_and_classic(ctx, devices):
    t.fsk_minmax_and_classic(ctx, devices, n=1 << 16)


def test_emu_cs8_and_cf32(ctx, devices):
    t.cs8_and_cf32(ctx, devices, n=1 << 16)


def test_emu_ragged_slots(ctx, devices):
    t.ragged_slots(ctx, devices, n=1 << 16)


def test_emu_chunk_and_segment_sizes(ctx, devices):
    t.chunk_and_segment_sizes(ctx, devices, n=1 << 16)


def test_emu_split_changed_mid_file(ctx, devices):
    t.split_changed_mid_file(ctx, devices, n=1 << 16)


def test_emu_spoiled_seeds(ctx, devices, monkeypatch):
    t.spoiled_seeds(ctx, devices, monkeypatch, n=1 << 16)


def test_emu_grabbing_chain(ctx, devices):
    t.grabbing_chain(ctx, devices, n=1 << 16)


def test_emu_decoders_and_analyzer(devices, monkeypatch):
    t.decoders_and_analyzer(devices, monkeypatch)


def test_emu_argument_errors(ctx, devices):
    t.argument_errors(ctx, devices)


def test_emu_set_split_does_not_split_chains(ctx, devices):
    t.set_split_does_not_split_chains(ctx, devices, n=1 << 16)


def test_emu_arena_overflow_exact_alloc(ctx, devices, monkeypatch):
    """The overflow rerun of a splitting chain with every buffer ending at its cap (-DR433B_EXACT_ALLOC)."""
    so = os.path.join(emu.HERE, "_build", "libr433b_emu_chain_split_exact.so")
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR433B_EXACT_ALLOC", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", so])
    monkeypatch.setenv("SIMT_GUARD", "back")  # read by the library's first allocation
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = so, None
    c = lib.Context()
    try:
        c.set_devices(devices)
        t.arena_overflow(c, devices, monkeypatch, n=1 << 16)
    finally:
        c.close()
        lib.LIB_PATH, lib._lib = old
