"""-m gpu: k_detect's single FM path (r433b_detect.cuh: fm_demand and the stage pass at the end of k_detect).  The walk
makes FM on demand for every filter: a filter the host cannot prove monotone (-Y ratio above 0.5) gets its windows in
order from the last exact state, also across the launches of a time-sliced batch.  Stage arrays are made by a pass of
their own after the walk, so a batch with stage arrays skips idle tiles like any other.  Every case compares with the
oracle (and with the compiled reference when it is present).  tests/test_emu_fm_on_demand.py runs the same bodies
under the SIMT emulator."""
import numpy as np
import pytest

import helpers
from oracle import refh
from rtl_433_b200 import lib, synth
from test_gpu_parity import check, ctx, devices, oracle_for, run_gpu  # noqa: F401  (fixtures)
from test_idle_skip import idle_heavy, run_skipping

pytestmark = pytest.mark.gpu

WRAPPING = 0.6  # -Y ratio above 0.5: the feedback coefficient is negative, the filter is not provably monotone
FSK_RATE = 1024000


def reference(stages, low_pass=0.0):
    """The compiled reference with the default decoders, or None when it is not present."""
    if not refh.available():
        return None
    r = refh.Ref(store_bitbuffers=False, store_stages=stages)
    r.register_defaults()
    if low_pass:
        r.set_fm_low_pass(low_pass)
    return r


def oracle_with(devices, stages, low_pass):
    o = oracle_for(devices, stages=stages)
    o.set_fm_low_pass(low_pass)
    return o


def wrapping_filter_on_cs16_fsk(ctx, devices):
    """cs16 2-FSK with the wrapping filter, both FSK pulse detectors, with and without stage arrays (run_gpu)."""
    streams = [synth.fsk_stream(500 + seed, n_samples=1 << 18, n_bursts=2) for seed in range(2)]
    o = oracle_with(devices, True, WRAPPING)
    r = reference(True, WRAPPING)
    ctx.set_fm_low_pass(WRAPPING)
    try:
        for fpdm, freq in ((lib.FPDM_AUTO, 868000000), (lib.FPDM_CLASSIC, 433920000)):
            gpu = run_gpu(ctx, streams, lib.FMT_CS16, FSK_RATE, freq, fpdm)
            for i, s in enumerate(streams):
                want = o.run(s, 4, FSK_RATE, freq, fpdm)
                assert any(p["type"] == 2 for p in want["packages"])
                check(gpu[i], want, f"wrapping cs16 fpdm {fpdm} stream {i}")
                if r:
                    check(gpu[i], r.run(s, 4, FSK_RATE, freq, fpdm), f"wrapping cs16 fpdm {fpdm} stream {i} vs reference")
    finally:
        ctx.set_fm_low_pass(0.0)


def test_wrapping_filter_on_cs16_fsk(ctx, devices):
    wrapping_filter_on_cs16_fsk(ctx, devices)


def wrapping_filter_across_time_slices(ctx, devices):
    """Time slices with the wrapping filter: the in-order FM of the next launch catches up from the filter state
    StreamState carried over, and the result is the oracle's."""
    streams = [synth.fsk_stream(510 + seed, n_samples=1 << 19, n_bursts=3) for seed in range(3)]
    o = oracle_with(devices, False, WRAPPING)
    refs = [o.run(s, 4, FSK_RATE, 868000000) for s in streams]
    assert all(any(p["type"] == 2 for p in ref["packages"]) for ref in refs)
    lens = [s.nbytes for s in streams]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    data = np.concatenate([s.view(np.uint8) for s in streams])
    ctx.set_fm_low_pass(WRAPPING)
    try:
        for groups in (3, 16):
            ctx.set_pipeline(groups)
            ctx.process(data, offsets, lib.FMT_CS16, FSK_RATE, 868000000)
            ctx.fetch()
            assert ctx.timing()["detect_launches"] > 1
            for i in range(len(streams)):
                got = helpers.gpu_stream_results(ctx, i)
                check(got, refs[i], f"wrapping, pipeline {groups} stream {i}")
    finally:
        ctx.set_pipeline(0)
        ctx.set_fm_low_pass(0.0)


def test_wrapping_filter_across_time_slices(ctx, devices):
    wrapping_filter_across_time_slices(ctx, devices)


def idle_heavy_streams_with_stage_arrays(ctx, devices):
    """A batch with stage arrays skips idle tiles, and its AM / FM stage arrays are the oracle's (and the reference's)."""
    streams = idle_heavy()
    lens = [s.nbytes for s in streams]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ctx.process(np.concatenate(streams), offsets, lib.FMT_CU8, 250000, 433920000, want_stages=True)
    ctx.fetch()
    tm = ctx.timing()
    o = oracle_for(devices, stages=True)
    r = reference(True)
    for i, s in enumerate(streams):
        got = helpers.gpu_stream_results(ctx, i)
        got["am"], got["fm"] = ctx.copy_stage(i, lens[i] // 2)
        assert len(got["fm"]) == lens[i] // 2
        want = o.run(s, 2)
        assert want["packages"] and len(want["am"]) == len(want["fm"]) == lens[i] // 2
        check(got, want, f"idle-heavy with stages, stream {i}")
        if r:
            check(got, r.run(s, 2), f"idle-heavy with stages, stream {i} vs reference")
    assert tm["idle_skipped"] > 0, tm


def test_idle_heavy_streams_with_stage_arrays(ctx, devices):
    idle_heavy_streams_with_stage_arrays(ctx, devices)


def idle_heavy_streams_with_a_wrapping_filter(ctx, devices):
    """Idle tiles are skipped with the wrapping filter too: the next FM window is made in order from the last exact
    state across the skipped tiles."""
    streams = idle_heavy()
    ctx.set_fm_low_pass(WRAPPING)
    try:
        got, tm = run_skipping(ctx, streams)
    finally:
        ctx.set_fm_low_pass(0.0)
    o = oracle_with(devices, False, WRAPPING)
    r = reference(False, WRAPPING)
    for i, s in enumerate(streams):
        want = o.run(s, 2)
        assert want["packages"]
        check(got[i], want, f"idle-heavy wrapping, stream {i}")
        if r:
            check(got[i], r.run(s, 2), f"idle-heavy wrapping, stream {i} vs reference")
    assert tm["idle_skipped"] > 0, tm


def test_idle_heavy_streams_with_a_wrapping_filter(ctx, devices):
    idle_heavy_streams_with_a_wrapping_filter(ctx, devices)
