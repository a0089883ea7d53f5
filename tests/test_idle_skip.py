"""-m gpu: k_detect's idle-tile skip (r433b_detect.cuh, idle_skip).  Noise tiles are ruled out from k_front's tile
summaries, and the exact noise floor behind a skipped run is recovered from the last skipped tile's AM (or, should
that fail, by walking the run again).  Results must be exactly those of the oracle (and of the compiled reference),
and the counters must show that the skip ran.  tests/test_emu_idle_skip.py runs the same bodies under the SIMT
emulator, once more with every skipped run walked again."""
import numpy as np
import pytest

import helpers
from oracle import refh
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices, oracle_for  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

RATE = 250000


def run_skipping(ctx, streams, block_bytes=0, lengths=None):
    """One cu8 batch without stage arrays: per-stream results and the timing counters."""
    lens = [s.nbytes for s in streams]
    assert all(n % 16 == 0 for n in lens)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    data = np.concatenate([s.view(np.uint8).ravel() for s in streams])
    ctx.process(data, offsets, lib.FMT_CU8, RATE, 433920000, lib.FPDM_AUTO, block_bytes, want_stages=False, lengths=lengths)
    ctx.fetch()
    return [helpers.gpu_stream_results(ctx, i) for i in range(len(streams))], ctx.timing()


def check(got, want, tag):
    d = helpers.compare_results(want, got, tag, stages=False)
    assert not d, "\n".join(d[:20])


def idle_heavy(n_samples=1 << 18):
    return [synth.ook_stream(300 + seed, n_samples=n_samples, n_bursts=1 + seed % 2) for seed in range(4)]


def idle_heavy_streams_match_the_oracle_and_the_reference(ctx, devices):
    streams = idle_heavy()
    got, tm = run_skipping(ctx, streams)
    o = oracle_for(devices, stages=False)
    for i, s in enumerate(streams):
        want = o.run(s, 2)
        assert want["packages"]
        check(got[i], want, f"idle-heavy stream {i}")
    if refh.available():
        r = refh.Ref(store_bitbuffers=False, store_stages=False)
        r.register_defaults()
        for i, s in enumerate(streams):
            check(got[i], r.run(s, 2), f"idle-heavy stream {i} vs reference")
    tiles = sum(len(s) // 2 // 2048 for s in streams)
    assert tm["idle_skipped"] > tiles // 2, tm
    return tm


def test_idle_heavy_streams_match_the_oracle_and_the_reference(ctx, devices):
    idle_heavy_streams_match_the_oracle_and_the_reference(ctx, devices)


def bursts_right_behind_a_skipped_run(ctx, devices):
    """The first pulse of a train starts at sample 0, 1 and 63 of a tile behind many noise tiles: the tracker's exact
    value in front of it comes from the resolution of the skipped run."""
    streams = []
    for k, off in enumerate((0, 1, 63, 2047)):
        pos = (40 + 3 * k) * 2048 + off
        streams.append(synth.ook_train_stream(400 + k, 24, n_samples=1 << 18, lead_us=pos * 1e6 / RATE))
    got, tm = run_skipping(ctx, streams)
    o = oracle_for(devices, stages=False)
    for i, s in enumerate(streams):
        want = o.run(s, 2)
        assert want["packages"]
        check(got[i], want, f"train behind a skipped run {i}")
    assert tm["idle_skipped"] >= 4 * 30, tm
    return tm


def test_bursts_right_behind_a_skipped_run(ctx, devices):
    bursts_right_behind_a_skipped_run(ctx, devices)


def ragged_lengths_and_small_blocks_with_skipping(ctx, devices):
    """Partial last tiles, and blocks of 8 tiles whose starts fall inside skipped runs."""
    base = synth.ook_stream(310, n_samples=1 << 18, n_bursts=1)
    streams = [base[:c].copy() for c in (2 * 16 * 4097, 2 * 131072 + 2 * 16 * 3, 2 * 8 * 99991 // 16 * 16, len(base))]
    o = oracle_for(devices, stages=False)
    for bb in (0, 32768):
        got, tm = run_skipping(ctx, streams, block_bytes=bb)
        for i, s in enumerate(streams):
            check(got[i], o.run(s, 2, block_bytes=bb), f"ragged {i} block {bb}")
        assert tm["idle_skipped"] > 0, tm


def test_ragged_lengths_and_small_blocks_with_skipping(ctx, devices):
    ragged_lengths_and_small_blocks_with_skipping(ctx, devices)


def time_slices_with_skipping(ctx, devices):
    """Pipelined time slices: a skipped run never crosses a slice end (the last tile of a launch is walked), and the
    carried state is the single-launch one."""
    streams = idle_heavy(1 << 19)
    o = oracle_for(devices, stages=False)
    refs = [o.run(s, 2) for s in streams]
    try:
        for groups in (3, 16):
            ctx.set_pipeline(groups)
            got, tm = run_skipping(ctx, streams)
            assert tm["detect_launches"] > 1
            assert tm["idle_skipped"] > 0, tm
            for i in range(len(streams)):
                check(got[i], refs[i], f"pipeline {groups} stream {i}")
    finally:
        ctx.set_pipeline(0)


def test_time_slices_with_skipping(ctx, devices):
    time_slices_with_skipping(ctx, devices)


def repairs_between_skipped_runs(devices, monkeypatch):
    """R433B_SPOIL_FRONT=3 spoils k_front's guess for lane 0 of every 7th tile: those tiles fail the hand-over check,
    end a skipped run and are repaired, and skipping resumes behind them."""
    streams = idle_heavy()
    monkeypatch.setenv("R433B_SPOIL_FRONT", "3")
    c = lib.Context(0)
    monkeypatch.delenv("R433B_SPOIL_FRONT")
    try:
        c.set_devices(devices)
        got, tm = run_skipping(c, streams)
    finally:
        c.close()
    o = oracle_for(devices, stages=False)
    for i, s in enumerate(streams):
        check(got[i], o.run(s, 2), f"spoil 3 stream {i}")
    tiles = sum(len(s) // 2 // 2048 for s in streams)
    assert tm["front_repairs"] >= tiles // 7 - len(streams), tm
    assert tm["idle_skipped"] > tiles // 3, tm


def test_repairs_between_skipped_runs(devices, monkeypatch):
    repairs_between_skipped_runs(devices, monkeypatch)
