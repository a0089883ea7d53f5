"""CPU: mixed batches under the SIMT emulator (tests/emu.py) -- the bodies of tests/test_mixed.py at smaller sizes, on
the kernels' own source: the class launches over their stream ranges, k_mixed_order and the slicers per rate, including
one arena overflow under the exact-allocation build."""
import os
import subprocess

import pytest

import emu
import test_mixed as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_per_stream_parity(ctx, devices):
    t.per_stream_parity(ctx, devices, n=1 << 16)


def test_emu_forced_fpdm_with_gates(ctx, devices):
    t.per_stream_parity(ctx, devices, n=1 << 16, gates=True, fpdm=lib.FPDM_MINMAX, analyze=False, reverse=True)


def test_emu_homogeneous_equals_process(ctx, devices):
    t.homogeneous(ctx, devices, n=1 << 16)


def test_emu_refusals(ctx, devices):
    t.refusals(ctx, devices)


def test_emu_arena_overflow_exact_alloc(devices, monkeypatch):
    """The overflow rerun with every buffer ending at its cap (-DR433B_EXACT_ALLOC)."""
    so = os.path.join(emu.HERE, "_build", "libr433b_emu_mixed_exact.so")
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
