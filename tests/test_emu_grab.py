"""CPU: k_grab and the grab plan under the SIMT emulator (tests/emu.py), with the bodies of the -m gpu tests in
tests/test_grab.py: every file name and byte against the compiled reference and the committed fingerprints."""
import pytest

import emu
import test_grab
from rtl_433_b200 import lib


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    old = (lib.LIB_PATH, lib._lib)
    emu.use()
    yield
    lib.LIB_PATH, lib._lib = old


@test_grab.needs_ref
@pytest.mark.parametrize("variant", ["plain", "gated", "parallel"])
def test_emu_modes_with_reference_decoders(variant):
    test_grab.modes_with_decoders(variant)


def test_emu_formats_pipeline_prior_and_pages():
    test_grab.formats_and_paths()


def test_emu_command_line_and_existing_names():
    test_grab.command_line_and_existing_names()


@test_grab.needs_ref
def test_emu_state_errors():
    test_grab.state_errors()
