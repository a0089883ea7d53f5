"""-m gpu: every overflow-and-rerun path gives what a run that did not overflow gives.

A context's package cap, pulse pool and event arena start at sizes that no small input reaches, and they only grow.
R433B_TEST_CAPS=pkg,pool,arena (read by r433b_create) starts a fresh context with small ones, so that small inputs take
each rerun path:
  * r433b_process_pulses: the event arena overflows in a later range after earlier ranges wrote, gated and ungated
    (slice_ranges slices every range again into a grown arena);
  * sequential IQ: package-cap, pulse-pool and event-arena overflow, alone and together (k_detect runs again from the
    reset state, k_slice2 again into a grown arena);
  * time-sliced IQ: an overflow in a middle slice, after which the whole batch is redone sequentially;
  * chained batches: the chunk that overflows starts and ends inside open packages; the rerun starts again from the
    chain's state and pulse trains as they were in front of the chunk.
Each case is compared with a fresh context with the default caps and, for IQ input, with the oracle; each asserts
from r433b_timing that the rerun happened.  One case needs no hook: a capture of back-to-back 1200-pulse packages
outgrows the default pulse pool of a one-stream batch.  tests/test_emu_slice_fuzz.py runs the hooked cases under the
SIMT emulator."""
import numpy as np
import pytest

import helpers
from oracle import orc
from rtl_433_b200 import lib, synth
import test_chain
import test_slice_fuzz
from test_oracle_vs_ref import random_train

OOK_RATE = 250000


def fresh(devices, monkeypatch=None, caps=None):
    if caps is not None:
        monkeypatch.setenv("R433B_TEST_CAPS", ",".join(str(int(c)) for c in caps))
    try:
        c = lib.Context(0)
    finally:
        if caps is not None:
            monkeypatch.delenv("R433B_TEST_CAPS")
    c.set_devices(devices)
    return c


def not_line_multiple(n):
    """A cap near n that is a multiple of 16 but not of 128: the warp whose range reaches it copies part of its lines."""
    return max(n // 128, 1) * 128 + 48


def results(ctx, n_streams):
    return [helpers.gpu_stream_results(ctx, s) for s in range(n_streams)]


def same(got, want, tag):
    for s, (g, w) in enumerate(zip(got, want)):
        d = helpers.compare_results(w, g, f"{tag} stream {s}", stages=False)
        assert not d, "\n".join(d[:20])


# ------------------------------------------------------------------------------------------------ cases ------

def short_packages(seed, per_run):
    """Short OOK and FSK packages of nominal symbol mixes, in the runs of test_slice_fuzz.RATE_RUNS: no pair comes near
    kStageWords, so every warp copies its lanes out of window and scratch -- the warp whose arena range reaches the
    cap copies the part below it."""
    rng = np.random.default_rng(seed)
    runs = []
    for rate in test_slice_fuzz.RATE_RUNS:
        r = []
        for _ in range(per_run):
            pulse, gap = random_train(rng, 0)
            n = int(rng.integers(1, 24))
            r.append(test_slice_fuzz._pd(rate, pulse[:n], gap[:n], int(rng.integers(1, 9000)) if rng.random() < 0.4 else 0))
        runs.append(r)
    return runs


def pulses_arena_overflow_in_a_later_range(devices, monkeypatch, per_run=40):
    runs = short_packages(31, per_run)
    ps = lib.Pulses()
    for s, r in enumerate(runs):
        for pd in r:
            ps.add(pd, stream=s)
    n_ranges = len(set(test_slice_fuzz.RATE_RUNS))
    for gates in (None, lib.default_gates(devices)):
        clean = fresh(devices)
        try:
            clean.set_gates(gates)
            clean.process_pulses(ps)
            res = clean.fetch()
            want = results(clean, len(runs))
            pk = res["packages"]
            rows = res["pairs"][pk["first_pair"] // res["n_devices"]]
            # bytes of the first range (the lowest rate: ranges are in rate order; stream i holds one rate)
            first = np.array([test_slice_fuzz.RATE_RUNS[int(s)] == min(test_slice_fuzz.RATE_RUNS) for s in pk["stream"]])
            b0, total = int(rows["bytes"][first].sum()), res["event_bytes"]
            want_gated = res["n_gated"]
        finally:
            clean.close()
        cap = not_line_multiple((b0 + total) // 2)
        assert b0 < cap < total and cap % 128, (b0, cap, total)
        c = fresh(devices, monkeypatch, (0, 0, cap))
        try:
            c.set_gates(gates)
            c.process_pulses(ps)
            res = c.fetch()
            assert c.timing()["slice_launches"] == 2 * n_ranges, c.timing()
            assert res["event_bytes"] == total and res["n_gated"] == want_gated
            assert (res["pairs"]["bytes"] <= test_slice_fuzz.STAGE_BYTES).all()
            test_slice_fuzz.check_pairs(c, res, n_ranges)
            same(results(c, len(runs)), want, f"arena cap {cap}, gates {'on' if gates else 'off'}")
        finally:
            c.close()
    ps.close()


@pytest.mark.gpu
def test_pulses_arena_overflow_in_a_later_range(monkeypatch):
    pulses_arena_overflow_in_a_later_range(lib.default_device_table(), monkeypatch, 400)


def iq_streams(n_streams=4, n_samples=1 << 18, seed=900):
    return [synth.ook_stream(seed + k, n_samples=n_samples, n_bursts=2)
            for k in range(n_streams)]


def run_iq(ctx, streams, pipeline):
    data = np.concatenate(streams)
    offsets = np.concatenate([[0], np.cumsum([s.nbytes for s in streams])]).astype(np.uint64)
    ctx.set_pipeline(pipeline)
    ctx.process(data, offsets, lib.FMT_CU8, OOK_RATE, 433920000)
    res = ctx.fetch()
    return res, results(ctx, len(streams)), ctx.timing()


KEPT = ("idle_skipped", "front_repairs", "front_redone", "idle_rewalks")


def sequential_iq_overflows(devices, monkeypatch, n_samples=1 << 18):
    streams = iq_streams(n_samples=n_samples)
    o = orc.Oracle(store_bitbuffers=False)
    o.add_devices(devices)
    want = [o.run(s, 2) for s in streams]
    o.close()
    clean = fresh(devices)
    try:
        res, got, tm0 = run_iq(clean, streams, 1)
        same(got, want, "default caps vs oracle")
        n_pkgs, pool, arena = res["n_packages"], int(res["packages"]["pulse_count"].sum()), res["event_bytes"]
    finally:
        clean.close()
    assert n_pkgs >= 8 and tm0["detect_launches"] == 1 and tm0["slice_launches"] == 1
    big = 1 << 24
    cases = {"packages": ((n_pkgs // 2, big, 0), 2, 1), "pool": ((0, pool // 2, 0), 2, 1),
             "arena": ((0, 0, not_line_multiple(arena // 2)), 1, 2),
             "all": ((n_pkgs // 3, pool // 3, not_line_multiple(arena // 3)), 2, 2)}
    for name, (caps, detects, slices) in cases.items():
        c = fresh(devices, monkeypatch, caps)
        try:
            _res, got, tm = run_iq(c, streams, 1)
            assert (tm["detect_launches"], tm["slice_launches"]) == (detects, slices), (name, tm)
            # the statistics describe the attempt that counted
            assert {k: tm[k] for k in KEPT} == {k: tm0[k] for k in KEPT}, name
            same(got, want, f"{name} overflow")
        finally:
            c.close()


@pytest.mark.gpu
def test_sequential_iq_overflows(monkeypatch):
    sequential_iq_overflows(lib.default_device_table(), monkeypatch)


def time_sliced_overflow_in_a_middle_slice(devices, monkeypatch, n_samples=1 << 18):
    streams = iq_streams(n_samples=n_samples, seed=910)
    o = orc.Oracle(store_bitbuffers=False)
    o.add_devices(devices)
    want = [o.run(s, 2) for s in streams]
    o.close()
    clean = fresh(devices)
    try:
        res, got, tm0 = run_iq(clean, streams, 4)
        same(got, want, "time-sliced, default caps vs oracle")
        pk = res["packages"].copy()  # a view of the context's host buffers
    finally:
        clean.close()
    assert tm0["detect_launches"] == 4
    cap = len(pk) // 2
    # the packages found in the first slice fit: the overflow happens in a later one
    slice_samples = -(-(n_samples // 4) // 2048) * 2048
    assert (pk["end_pos"] < slice_samples).sum() < cap < len(pk)
    c = fresh(devices, monkeypatch, (cap, 1 << 24, 0))
    try:
        _res, got, tm = run_iq(c, streams, 4)
        # the time-sliced attempt is abandoned and the batch redone in ONE sequential launch
        assert tm["detect_launches"] == 1 and tm["slice_launches"] == 1, tm
        same(got, want, "time-sliced overflow redone sequentially")
    finally:
        c.close()


@pytest.mark.gpu
def test_time_sliced_overflow_in_a_middle_slice(monkeypatch):
    time_sliced_overflow_in_a_middle_slice(lib.default_device_table(), monkeypatch)


BLOCK = 4096  # bytes of cu8: 2048 samples


def dense_file(seed=950, sparse_blocks=8, dense_blocks=64, tail_blocks=8):
    """cu8: a sparse first chunk, a dense second one, a third; a long train crosses each chunk boundary."""
    rng = np.random.default_rng(seed)
    spb = BLOCK // 2
    b1, b2 = sparse_blocks * spb, (sparse_blocks + dense_blocks) * spb
    n = (sparse_blocks + dense_blocks + tail_blocks) * spb
    x = rng.standard_normal(2 * n, dtype=np.float32) * np.float32(2.0) + np.float32(127.5)

    def burst():  # a short PWM burst, about 6 ms
        return [(float(rng.choice([250, 750])), 1) if k % 2 == 0 else (500.0, 0) for k in range(47)] + [(0.0, 0)]

    def put(pos, seg):
        m = synth._render_ook(seg, OOK_RATE).astype(np.float32) * np.float32(rng.uniform(60, 100))
        ph = rng.uniform(0, 2 * np.pi) + 2 * np.pi * rng.uniform(-40e3, 40e3) / OOK_RATE * np.arange(len(m))
        x[2 * pos:2 * (pos + len(m)):2] += m * np.cos(ph).astype(np.float32)
        x[2 * pos + 1:2 * (pos + len(m)) + 1:2] += m * np.sin(ph).astype(np.float32)
        return pos + len(m)

    train = [(200.0, 1), (200.0, 0)] * 150  # 150 pulses, 24,000 samples
    put(2500, burst())
    put(b1 - 6000, train)                   # open across the first boundary
    pos = b1 + 20000
    while pos < b2 - 30000:                 # dense: a burst every ~15 ms
        pos = put(pos, burst()) + 3000
    put(b2 - 6000, train)                   # open across the second boundary
    return np.clip(np.rint(x), 0, 255).astype(np.uint8), (sparse_blocks, sparse_blocks + dense_blocks)


def chained_overflow_inside_open_packages(devices, monkeypatch, pipeline):
    x, cuts = dense_file()
    chunks = test_chain.cut(x, BLOCK, cuts)
    clean = fresh(devices)
    try:
        want = test_chain.run_uncut(clean, [x], lib.FMT_CU8, OOK_RATE, block_bytes=BLOCK)[0]
    finally:
        clean.close()
    spb = BLOCK // 2
    b1, b2 = cuts[0] * spb, cuts[1] * spb
    pk = want["packages"]
    spans = lambda b: any(p["offset"] < b < p["offset"] + int(p["pulse"].sum() + p["gap"].sum()) for p in pk)  # noqa: E731
    assert spans(b1) and spans(b2), "no package open across a chunk boundary"
    in_first = sum(1 for p in pk if p["offset"] + int(p["pulse"].sum() + p["gap"].sum()) < b1)
    in_second = len(pk) - in_first
    assert in_second >= 4 * max(in_first, 1), (in_first, in_second)
    cap = in_first + 2
    c = fresh(devices, monkeypatch, (cap, 0, 0))
    try:
        c.set_pipeline(pipeline)
        got = test_chain._empty()
        launches = []
        with lib.Chain(c, 1) as chain:
            for j, ch in enumerate(chunks):
                data, offsets, lens = test_chain._pack([ch])
                c.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=BLOCK, lengths=lens, chain=chain,
                          last=[int(j == len(chunks) - 1)])
                res = c.fetch()
                launches.append(c.timing()["detect_launches"])
                test_chain._add(got, c, res, 0, len(ch) // 2, False)
        got = test_chain._finish(got, False)
    finally:
        c.close()
    if pipeline == 1:
        assert launches == [1, 2, 1], launches      # the dense chunk ran twice
    else:
        assert launches[0] == launches[2] == 4 and launches[1] == 1, launches  # ... redone sequentially
    test_chain.check(got, want, f"chained overflow, pipeline {pipeline}", stages=False)


@pytest.mark.gpu
@pytest.mark.parametrize("pipeline", [1, 4])
def test_chained_overflow_inside_open_packages(monkeypatch, pipeline):
    chained_overflow_inside_open_packages(lib.default_device_table(), monkeypatch, pipeline)


@pytest.mark.gpu
def test_back_to_back_1200_pulse_packages_outgrow_the_default_pool():
    """No hook: a one-stream batch has a pool of (16 + 1024) * 128 ints, and 120 packages of 1200 pulses need more.
    Each train is a little longer than PD_MAX_PULSES, so that it gives one full package whatever its first pulses do."""
    devices = lib.default_device_table()
    rng = np.random.default_rng(960)
    seg = []
    for _ in range(120):
        for _p in range(1210):
            seg += [(float(rng.integers(80, 120)), 1), (float(rng.integers(80, 120)), 0)]  # 20 .. 30 samples each
        seg.append((12000.0, 0))  # 12 ms between packages
    seg = [(8000.0, 0)] + seg
    m = synth._render_ook(seg, OOK_RATE).astype(np.float32) * np.float32(80.0)
    n = len(m) + 4096
    x = rng.standard_normal(2 * n, dtype=np.float32) * np.float32(2.0) + np.float32(127.5)
    ph = 2 * np.pi * 20e3 / OOK_RATE * np.arange(len(m))
    x[0:2 * len(m):2] += m * np.cos(ph).astype(np.float32)
    x[1:2 * len(m) + 1:2] += m * np.sin(ph).astype(np.float32)
    x = np.clip(np.rint(x), 0, 255).astype(np.uint8)[:n // 8 * 16]
    assert x.nbytes > 7_000_000
    o = orc.Oracle(store_bitbuffers=False)
    o.add_devices(devices)
    want = o.run(x, 2)
    o.close()
    assert sum(1 for p in want["packages"] if p["num_pulses"] == 1200) >= 115
    assert sum(p["pulse_count"] for p in want["packages"]) > (16 + 1024) * 128
    c = fresh(devices)
    try:
        c.process(x, np.array([0, x.nbytes], np.uint64), lib.FMT_CU8, OOK_RATE, 433920000)
        c.fetch()
        assert c.timing()["detect_launches"] == 2, c.timing()
        same([helpers.gpu_stream_results(c, 0)], [want], "1200-pulse packages")
    finally:
        c.close()
