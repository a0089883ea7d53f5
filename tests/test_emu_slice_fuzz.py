"""CPU: the bodies of tests/test_slice_fuzz.py and tests/test_overflow.py under the SIMT emulator (tests/emu.py), smaller.

The fuzz runs on the regular emulated build and on the one with an 8-word write-combining window
(test_emu_small_window.py), where nearly every event slides the window.  The overflow cases run on a build whose
device buffers end exactly at their caps, behind a guard page (SIMT_GUARD=back): a k_slice2 copy that writes one word
past the event arena's cap faults there instead of landing in the growth slack."""
import os
import subprocess

import pytest

import emu
import test_emu_small_window
from rtl_433_b200 import lib


@pytest.fixture
def emulated():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


@pytest.fixture
def small_window():
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = test_emu_small_window.build_small_window(), None
    yield
    lib.LIB_PATH, lib._lib = old


EXACT_SO = os.path.join(emu.HERE, "_build", "libr433b_emu_exact.so")


@pytest.fixture(scope="module")
def exact_so():
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    os.makedirs(os.path.dirname(EXACT_SO), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR433B_EXACT_ALLOC", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", EXACT_SO])
    return EXACT_SO


@pytest.fixture
def exact_alloc(exact_so, monkeypatch):
    """The emulated build with -DR433B_EXACT_ALLOC, its buffers ending right at the rear guard page."""
    monkeypatch.setenv("SIMT_GUARD", "back")  # read by the library's first allocation
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = EXACT_SO, None
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_random_packages_through_k_slice2(emulated):
    import test_slice_fuzz
    test_slice_fuzz.slice_fuzz(7, [33, 45, 65], [1, 3, 5], 200, 30000)


def test_emu_small_window_random_packages_through_k_slice2(small_window):
    import test_slice_fuzz
    test_slice_fuzz.slice_fuzz(8, [33, 45, 65], [1, 3, 5], 200, 30000)


def test_emu_pulses_arena_overflow_in_a_later_range(exact_alloc, monkeypatch):
    import test_overflow
    test_overflow.pulses_arena_overflow_in_a_later_range(lib.default_device_table(), monkeypatch)


def test_emu_sequential_iq_overflows(exact_alloc, monkeypatch):
    import test_overflow
    test_overflow.sequential_iq_overflows(lib.default_device_table(), monkeypatch)


def test_emu_time_sliced_overflow_in_a_middle_slice(exact_alloc, monkeypatch):
    import test_overflow
    test_overflow.time_sliced_overflow_in_a_middle_slice(lib.default_device_table(), monkeypatch)


@pytest.mark.parametrize("pipeline", [1, 4])
def test_emu_chained_overflow_inside_open_packages(exact_alloc, monkeypatch, pipeline):
    import test_overflow
    test_overflow.chained_overflow_inside_open_packages(lib.default_device_table(), monkeypatch, pipeline)
