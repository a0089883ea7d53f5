"""CPU: k_slice2 with its write-combining window shrunk to one 32-byte sector (R4_SLICE_WINDOW=8) under the SIMT
emulator.  Events of more than a few words then slide the window, their header is patched into words already flushed
to the scratch, and gated or cleared events roll the window back below its base; the slicer parity cases, gates off
and on, must still give the oracle's (and the reference's) events."""
import os
import subprocess

import pytest

import emu
from rtl_433_b200 import lib

SMALL_WINDOW_SO = os.path.join(emu.HERE, "_build", "libr433b_emu_w8.so")


def build_small_window():
    """emu.build()'s library, with an 8-word window, beside the regular emulated build."""
    csrc = os.path.join(emu.ROOT, "rtl_433_b200", "csrc")
    os.makedirs(os.path.dirname(SMALL_WINDOW_SO), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-DR433B_SIMT_EMU",
                           "-DR4_SLICE_WINDOW=8", "-I" + os.path.join(emu.HERE, "simt"), "-x", "c++",
                           os.path.join(csrc, "r433b_api.cu"), "-o", SMALL_WINDOW_SO])
    return SMALL_WINDOW_SO


@pytest.fixture(scope="module", autouse=True)
def small_window_library():
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = build_small_window(), None
    yield
    lib.LIB_PATH, lib._lib = old


from test_gpu_parity import (ctx, devices,  # noqa: E402,F401  (fixtures)
                             test_custom_piwm_raw_and_nrzs_devices, test_ook_1200_pulse_end_of_package,
                             test_ook_cu8_default_devices, test_fsk_cs16_minmax_and_classic)
import test_gates  # noqa: E402
import test_pulse_io  # noqa: E402


def test_small_window_gated_run_is_the_filtered_ungated_run():
    test_gates.gated_run_is_the_filtered_ungated_run()


@test_pulse_io.needs_ref
def test_small_window_loaded_packages_through_k_slice2():
    test_pulse_io.loaded_packages_through_k_slice2()
