"""-m gpu: segmented replay of mixed batches (include/r433b.h: r433b_process_mixed under r433b_set_split).  Every case
runs a mixed batch unsplit and split in one context and compares them with nothing relaxed: every package field (seq,
offset, end_pos and block included), the pulse and gap widths, every pair and event, the stream digests, every
pulse_data_t field and sample_file_pos, the analyzer text where asked, and the `-S all` grab plan with its bytes.  Where
it is cheap, each file alone through r433b_process() is the reference too.  Each case also asserts from r433b_timing
that it took the split path: more segments than streams, at most one rewalk per segment past a stream's first, the
unsplit run's classes, between one and L launches per pass and round (L: the unsplit run's launches), and no
k_mixed_order.  tests/test_emu_mixed_split.py runs the same bodies, smaller, under the SIMT emulator."""
import ctypes as C

import numpy as np
import pytest

import test_mixed as t
import test_split as ts
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BLOCK = t.BLOCK  # 16384 bytes: 8192 cu8 / cs8 samples, 4096 cs16 samples per block


def run(ctx, items, split=0, warmup=1, fpdm=lib.FPDM_AUTO, analyze=False, on_device=False, reverse=False):
    """One mixed batch of `items` (test_mixed.corpus's form) -> snapshots per stream, the grab, the timing."""
    data, offsets, lens = t._pack(items, reverse)
    keep = None
    if on_device:
        import torch
        keep = torch.from_numpy(data).cuda()
        data = keep.data_ptr()
    ctx.set_split(split, warmup)
    try:
        ctx.process_mixed(data, offsets, [x[2] for x in items], [x[3] for x in items], [x[4] for x in items],
                          lengths=lens, fpdm_mode=fpdm, data_on_device=on_device, block_bytes=BLOCK)
    finally:
        ctx.set_split(0)
    tm = ctx.timing()
    res = ctx.fetch()
    if analyze:
        ctx.analyze()
    out = {"snaps": [t._drop_positions(t.snapshot(ctx, res, i, analyze)) for i in range(len(items))], "tm": tm}
    plan = ctx.grab_plan(lib.GRAB_ALL)
    out["grab"] = (plan.tobytes(), ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes() if len(plan) else b"",
                   ctx.grab_tail()[1].tobytes())
    del keep
    return out


def check_split(tm, unsplit, n_streams, tag):
    """r433b_timing of a split mixed batch against the same batch unsplit."""
    assert tm["split_segments"] > n_streams, (tag, tm)
    assert tm["split_rewalks"] <= tm["split_segments"] - n_streams, (tag, tm)
    assert tm["mixed_classes"] == unsplit["mixed_classes"], (tag, tm, unsplit)
    L = unsplit["detect_launches"]
    assert 2 + tm["split_rounds"] <= tm["detect_launches"] <= L * (2 + tm["split_rounds"]), (tag, tm, L)
    assert tm["front_launches"] == tm["detect_launches"], (tag, tm)
    assert tm["mixed_order_ms"] == 0, (tag, tm)


def compare(ctx, items, split, warmup=1, alone=None, tag="", **kw):
    """Split against unsplit in one context (and against `alone`, the files alone); -> split timing, unsplit run."""
    want = run(ctx, items, **kw)
    assert want["tm"]["split_segments"] == 0, want["tm"]
    assert sum(len(s["headers"]) for s in want["snaps"]) > 3, f"{tag}: nothing detected, nothing checked"
    got = run(ctx, items, split, warmup, **kw)
    t.same(got["snaps"], want["snaps"], items, tag)
    assert got["grab"] == want["grab"], f"{tag}: -S all grab differs"
    if alone is not None:
        t.same(got["snaps"], alone, items, tag + " vs alone")
    check_split(got["tm"], want["tm"], len(items), tag)
    return got["tm"], want


def segments(items, split):
    """Segments per stream of an explicit segment size: blocks of the bytes after conversion (cf32 -> cs16)."""
    out = []
    for _, x, fmt, *_ in items:
        n = x.view(np.uint8).size // 8 * 4 if fmt == lib.FMT_CF32 else x.view(np.uint8).size
        blocks = -(-n // BLOCK)
        out.append(-(-blocks // split) if blocks > split else 1)
    return out


# ------------------------------------------------------------------------------------------------------- cases ------

def corpus_parity(ctx, devices, n=1 << 17, sizes=((1, 1), (2, 1), (2, 2), (3, 2), (lib.SPLIT_AUTO, 1))):
    """test_mixed's corpus (the empty file, the one shorter than a block, cf32, the 868 / 915 MHz cs16 pair) at several
    segment and warm-up sizes and with SPLIT_AUTO, against the unsplit batch and every file alone."""
    items = t.corpus(n)
    want = t.alone(ctx, items, analyze=True)
    for seg, warm in sizes:
        tm, _ = compare(ctx, items, seg, warm, alone=want, analyze=True, tag=f"segment {seg} warm-up {warm}")
        if seg != lib.SPLIT_AUTO:
            assert tm["split_segments"] == sum(segments(items, seg)), tm


def device_input(ctx, devices, n=1 << 17):
    """Device-resident input: cf32 converted into the second buffer, so its class is launched once per buffer."""
    items = t.corpus(n)
    want = t.alone(ctx, items)
    tm, unsplit = compare(ctx, items, 2, alone=want, on_device=True, tag="device input")
    assert unsplit["tm"]["detect_launches"] == unsplit["tm"]["mixed_classes"] + 1, unsplit["tm"]


def descending_offsets(ctx, devices, n=1 << 17):
    items = t.corpus(n)
    compare(ctx, items, 2, alone=t.alone(ctx, items), reverse=True, tag="descending offsets")


def gates_and_fpdm(ctx, devices, n=1 << 17, modes=(lib.FPDM_CLASSIC, lib.FPDM_MINMAX)):
    items = t.corpus(n)
    ctx.set_gates(lib.default_gates(devices))
    try:
        for fpdm in modes:
            compare(ctx, items, 2, alone=t.alone(ctx, items, fpdm), fpdm=fpdm, tag=f"gates, fpdm {fpdm}")
    finally:
        ctx.set_gates(None)


def open_items(n_segs):
    """Packages open across segment starts in four classes (two blocks per segment, one of warm-up): an OOK cu8 stream
    whose trains begin inside the warm-ups (seeds accepted), an OOK cs8 stream whose trains begin in front of them
    (rejected), FSK cu8 and cs16 streams with bursts all over."""
    seg = 2 * BLOCK // 2  # cu8 samples per segment
    inside = ts.trains_at(1200, [k * seg - 1500 for k in range(1, n_segs)], n_segs * seg)
    before = ts.trains_at(1201, [k * seg - BLOCK // 2 - 1500 for k in range(1, n_segs)], n_segs * seg, n_pulses=120)
    return [("ook_cu8_inside", inside, lib.FMT_CU8, 250000, 433920000),
            ("ook_cs8_before", before ^ 0x80, lib.FMT_CS8, 250000, 315000000),
            ("fsk_cu8", synth.fsk_burst_stream(1202, 64, n_samples=n_segs * seg, rate=1024000, cu8=True), lib.FMT_CU8,
             1024000, 868000000),
            ("fsk_cs16", ts.fsk(1203, n_segs * seg // 2), lib.FMT_CS16, 1024000, 868000000)]


def open_packages(ctx, devices, n_segs=8):
    """Seeds accepted and rejected in several classes at once, FM on (the default devices include FSK ones); again with
    a wrapping FM low-pass and at a non-default level point."""
    items = open_items(n_segs)
    tm, _ = compare(ctx, items, 2, 1, alone=t.alone(ctx, items), tag="open packages")
    assert 0 < tm["split_rewalks"] < tm["split_segments"] - len(items), tm
    assert tm["mixed_classes"] == 4, tm
    ctx.set_fm_low_pass(ts.WRAPPING)
    try:
        compare(ctx, items, 2, 1, alone=t.alone(ctx, items), tag="open packages, wrapping low-pass")
    finally:
        ctx.set_fm_low_pass(0.0)
    ctx.set_levels(1, -30.0, -12.1442, 9.0)
    try:
        compare(ctx, items, 2, 1, alone=t.alone(ctx, items), tag="open packages, magnitude, level -30")
    finally:
        ctx.set_levels()


def spoiled_seeds(devices, monkeypatch, n=1 << 17, split=2):
    """R433B_SPOIL_SEED=1: every seed is rejected.  Every segment past a stream's first is walked again, and the rounds
    are the most segments of one stream less one: the classes share their rounds.  (One-block segments of this corpus
    meet a known defect of the rewalk that one-format batches share, DESIGN §10.)"""
    monkeypatch.setenv("R433B_SPOIL_SEED", "1")
    c = lib.Context()
    try:
        c.set_devices(devices)
        items = t.corpus(n)
        tm, _ = compare(c, items, split, tag="spoiled seeds")
        segs = segments(items, split)
        assert tm["split_segments"] == sum(segs), tm
        assert tm["split_rewalks"] == tm["split_segments"] - len(items), tm
        assert tm["split_rounds"] == max(segs) - 1, (tm, segs)
    finally:
        c.close()


def arena_overflow(devices, monkeypatch, n=1 << 16):
    """Package and pool arenas far too small: the split schedule grows them and reruns from pass 0; the results equal
    the files alone and the split run with room, and the attempts that overflowed count in detect_launches."""
    items = t.corpus(n)
    c = lib.Context()
    try:
        c.set_devices(devices)
        want = t.alone(c, items)
        roomy = run(c, items, 2)
    finally:
        c.close()
    monkeypatch.setenv("R433B_TEST_CAPS", "4,64,256")
    c = lib.Context()
    try:
        c.set_devices(devices)
        got = run(c, items, 2)
    finally:
        c.close()
    t.same(got["snaps"], want, items, "overflow")
    t.same(got["snaps"], roomy["snaps"], items, "overflow vs room")
    assert got["grab"] == roomy["grab"]
    assert got["tm"]["split_segments"] == roomy["tm"]["split_segments"], got["tm"]
    assert got["tm"]["detect_launches"] > roomy["tm"]["detect_launches"], (got["tm"], roomy["tm"])
    assert got["tm"]["mixed_order_ms"] == 0, got["tm"]


def grab_vs_reference(ctx, devices, on_device=False):
    """test_mixed's grabber case at the reference's block size with one-block segments: equal to the stock reference's
    `rtl_433 -S all -r ...` (or tests/golden/grab_mixed.json where it is not built)."""
    ctx.set_split(1)
    try:
        t.grab_vs_reference(ctx, devices, on_device)
        tm = ctx.timing()
    finally:
        ctx.set_split(0)
    assert tm["split_segments"] > len(t.grab_case()), tm
    assert tm["mixed_order_ms"] == 0, tm


def homogeneous(ctx, devices, n=1 << 17, split=2):
    """One format through r433b_process_mixed split equals r433b_process split: digests and grabs."""
    items = [x for x in t.corpus(n) if x[2] == lib.FMT_CU8 and x[3] == 250000]
    data, offsets, lens = t._pack(items)

    def grab():
        plan = ctx.grab_plan(lib.GRAB_ALL)
        return (plan.tobytes(), ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes(),
                ctx.grab_tail()[1].tobytes())

    ctx.set_split(split)
    try:
        ctx.process(data, offsets, lib.FMT_CU8, 250000, 433920000, lib.FPDM_AUTO, BLOCK, lengths=lens)
        ctx.fetch()
        want_tm = ctx.timing()
        want = [ctx.stream_digest(i) for i in range(len(items))], grab()
        ctx.process_mixed(data, offsets, [lib.FMT_CU8] * len(items), [250000] * len(items), [433920000] * len(items),
                          lengths=lens, block_bytes=BLOCK)
        ctx.fetch()
        tm = ctx.timing()
        got = [ctx.stream_digest(i) for i in range(len(items))], grab()
    finally:
        ctx.set_split(0)
    assert got == want
    assert tm["split_segments"] == want_tm["split_segments"] > len(items), (tm, want_tm)
    assert tm["split_rounds"] == want_tm["split_rounds"] and tm["split_rewalks"] == want_tm["split_rewalks"], tm
    assert tm["detect_launches"] == want_tm["detect_launches"] == 2 + tm["split_rounds"], (tm, want_tm)
    assert tm["mixed_classes"] == 1 and tm["mixed_order_ms"] == 0, tm


def stays_unsplit(ctx, devices, n=1 << 16):
    """A mixed batch with no stream of two segments runs the unsplit schedule with splitting on, and stage arrays are
    still refused."""
    items = t.corpus(n)
    want = run(ctx, items)
    got = run(ctx, items, 64)
    assert got["tm"]["split_segments"] == 0, got["tm"]
    assert got["tm"]["detect_launches"] == want["tm"]["detect_launches"], got["tm"]
    t.same(got["snaps"], want["snaps"], items, "no stream of two segments")
    assert got["grab"] == want["grab"]
    data, offsets, lens = t._pack(items[:4])
    b = lib.Batch(data.ctypes.data, np.ascontiguousarray(offsets, np.uint64).ctypes.data_as(C.POINTER(C.c_uint64)),
                  4, 0, 0, 0, lib.FPDM_AUTO, BLOCK, 0, 1, None)
    f = (lib.StreamFormat * 4)(*[lib.StreamFormat(x[2], x[3], x[4]) for x in items[:4]])
    ctx.set_split(1)
    try:
        assert ctx.L.r433b_process_mixed(ctx.h, C.byref(b), f) == -1
    finally:
        ctx.set_split(0)
    t.same(run(ctx, items)["snaps"], want["snaps"], items, "after the refusal")


def many_streams_auto(ctx, devices):
    """SPLIT_AUTO with more streams than resident warps runs unsplit: 5000 short or empty streams of four classes
    beside one long one."""
    long_ = t.corpus(1 << 17)[0]
    short = [("short", long_[1][:32 * (k % 3)], f, r, q) for k, (f, r, q) in
             zip(range(4999), [(lib.FMT_CU8, 250000, 433920000), (lib.FMT_CS16, 1024000, 868000000),
                               (lib.FMT_CS8, 250000, 315000000), (lib.FMT_CU8, 2048000, 433920000)] * 1250)]
    items = [long_] + short
    data, offsets, lens = t._pack(items)
    fmts, rates, freqs = [x[2] for x in items], [x[3] for x in items], [x[4] for x in items]
    ctx.process_mixed(data, offsets, fmts, rates, freqs, lengths=lens, block_bytes=BLOCK)
    ctx.fetch()
    want = [ctx.stream_digest(i) for i in range(len(items))]
    ctx.set_split(lib.SPLIT_AUTO)
    try:
        ctx.process_mixed(data, offsets, fmts, rates, freqs, lengths=lens, block_bytes=BLOCK)
    finally:
        ctx.set_split(0)
    assert ctx.timing()["split_segments"] == 0, ctx.timing()
    ctx.fetch()
    assert [ctx.stream_digest(i) for i in range(len(items))] == want


# ------------------------------------------------------------------------------------------------------- tests ------

def test_corpus_parity(ctx, devices):
    corpus_parity(ctx, devices)


def test_device_input(ctx, devices):
    device_input(ctx, devices)


def test_descending_offsets(ctx, devices):
    descending_offsets(ctx, devices)


def test_gates_and_fpdm(ctx, devices):
    gates_and_fpdm(ctx, devices)


def test_open_packages(ctx, devices):
    open_packages(ctx, devices)


def test_spoiled_seeds(devices, monkeypatch):
    spoiled_seeds(devices, monkeypatch)


def test_arena_overflow(devices, monkeypatch):
    arena_overflow(devices, monkeypatch)


@pytest.mark.parametrize("on_device", [False, True])
def test_grab_vs_reference(ctx, devices, on_device):
    grab_vs_reference(ctx, devices, on_device)


def test_homogeneous_equals_process(ctx, devices):
    homogeneous(ctx, devices)


def test_stays_unsplit(ctx, devices):
    stays_unsplit(ctx, devices)


def test_many_streams_auto(ctx, devices):
    many_streams_auto(ctx, devices)
