"""CPU: tests/test_compact_events.py under the SIMT emulator (tests/emu.py), the write-combining window at its
regular size and shrunk to one sector (tests/test_emu_small_window.py's build)."""
import pytest

import emu
import test_compact_events as t
from rtl_433_b200 import lib
from test_emu_small_window import build_small_window


@pytest.fixture(scope="module", params=["window16", "window8"], autouse=True)
def emulated_library(request):
    old = (lib.LIB_PATH, lib._lib)
    lib.LIB_PATH, lib._lib = (emu.build() if request.param == "window16" else build_small_window()), None
    yield
    lib.LIB_PATH, lib._lib = old


def test_emu_custom_devices_match_the_oracle():
    t.custom_devices_match_the_oracle()


def test_emu_default_devices_on_the_edge_cases():
    t.default_devices_match()


def test_emu_stream_digest_hashes_the_long_form():
    t.stream_digest_hashes_the_long_form()
