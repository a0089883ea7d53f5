"""CPU: the body of tests/test_slice_layout.py under the SIMT emulator, on a build whose device buffers end exactly
at their caps in front of a guard page (-DR433B_EXACT_ALLOC, SIMT_GUARD=back): a k_bucket_scatter or k_slice2 access
past the computed size of the width copy faults there.  The build has a file of its own, so that test processes
running next to tests/test_emu_slice_fuzz.py never load a library the other one is still writing."""
import os
import subprocess

import pytest

import emu
from rtl_433_b200 import lib

EXACT_SO = os.path.join(emu.HERE, "_build", "libr433b_emu_exact_layout.so")


@pytest.fixture(scope="module")
def exact_alloc_so():
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    os.makedirs(os.path.dirname(EXACT_SO), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR433B_EXACT_ALLOC", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", EXACT_SO])
    return EXACT_SO


def test_emu_sorted_groups_and_interleaved_widths(exact_alloc_so, monkeypatch):
    import test_slice_layout
    monkeypatch.setenv("SIMT_GUARD", "back")  # read by the library's first allocation
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = exact_alloc_so, None
    try:
        test_slice_layout.slice_layout(11)
    finally:
        lib.LIB_PATH, lib._lib = old
