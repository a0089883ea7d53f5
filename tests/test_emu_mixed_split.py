"""CPU: segmented replay of mixed batches under the SIMT emulator (tests/emu.py) -- the bodies of
tests/test_mixed_split.py at smaller sizes, on the kernels' own source: the class launches of every pass and round over
one launch view, the merge in internal order and the slicers per rate, including one arena overflow under the
exact-allocation build.  The case with more streams than resident warps stays on the GPU."""
import os
import subprocess

import pytest

import emu
import test_mixed_split as t
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_corpus_parity(ctx, devices):
    t.corpus_parity(ctx, devices, n=1 << 16, sizes=((1, 1), (3, 2), (lib.SPLIT_AUTO, 1)))


def test_emu_descending_offsets(ctx, devices):
    t.descending_offsets(ctx, devices, n=1 << 16)


def test_emu_gates_and_fpdm(ctx, devices):
    t.gates_and_fpdm(ctx, devices, n=1 << 16, modes=(lib.FPDM_MINMAX,))


def test_emu_open_packages(ctx, devices):
    t.open_packages(ctx, devices, n_segs=4)


def test_emu_spoiled_seeds(devices, monkeypatch):
    t.spoiled_seeds(devices, monkeypatch, n=1 << 16, split=2)


def test_emu_homogeneous_equals_process(ctx, devices):
    t.homogeneous(ctx, devices, n=1 << 16)


def test_emu_stays_unsplit(ctx, devices):
    t.stays_unsplit(ctx, devices, n=1 << 16)


def test_emu_arena_overflow_exact_alloc(devices, monkeypatch):
    """The overflow rerun from pass 0 with every buffer ending at its cap (-DR433B_EXACT_ALLOC)."""
    so = os.path.join(emu.HERE, "_build", "libr433b_emu_mixed_split_exact.so")
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
