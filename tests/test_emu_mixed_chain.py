"""CPU: mixed batches on chains under the SIMT emulator (tests/emu.py) -- the bodies of tests/test_mixed_chain.py at
smaller sizes, on the kernels' own source: the gather of the slots' state into internal order, the class launches,
k_mixed_order with the carried start seq, the scatter back to the slots and the grabber's ring appends per source,
including one arena overflow under the exact-allocation build."""
import os
import subprocess

import pytest

import emu
import test_mixed_chain as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_corpus_parity(ctx, devices):
    t.corpus_parity(ctx, devices, n=1 << 16, blocks=3, analyze=False)


def test_emu_forced_fpdm_with_gates_descending(ctx, devices):
    t.corpus_parity(ctx, devices, n=1 << 16, blocks=1, gates=True, fpdm=lib.FPDM_MINMAX, analyze=False, reverse=True)


def test_emu_order_changes_between_calls(ctx, devices):
    t.order_changes(ctx, devices, n=1 << 16)


def test_emu_carried_state(ctx, devices):
    t.carried_state(ctx, devices, n=1 << 16)


def test_emu_spoiled_front(devices, monkeypatch):
    t.spoiled_front(devices, monkeypatch, n=1 << 16)


def test_emu_one_format_equals_process_chained(ctx, devices):
    t.one_format_equals_chained(ctx, devices, n=1 << 16)


def test_emu_split_chain_runs_unsplit(ctx, devices):
    t.split_chain_unsplit(ctx, devices, n=1 << 16)


def test_emu_grabbing_chain(ctx):
    t.grabbing_chain(ctx, n=1 << 19)


def test_emu_refusals(ctx, devices):
    t.refusals(ctx, devices)


def test_emu_arena_overflow_exact_alloc(devices, monkeypatch):
    """The overflow rerun from the carried state with every buffer ending at its cap (-DR433B_EXACT_ALLOC)."""
    so = os.path.join(emu.HERE, "_build", "libr433b_emu_mixed_chain_exact.so")
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
