"""-m gpu: segmented replay (include/r433b.h: r433b_set_split).  Every case runs a batch unsplit and split in the same
context and compares them with nothing relaxed: every package field (seq and end_pos included), the pulse and gap
widths, every event of every (package, device) pair, the stream digests, and where asked the analyzer text and the
`-S all` grab plan with its bytes.  Each case also asserts from r433b_timing that it took the path it is about.
tests/test_emu_split.py runs the same bodies, smaller, under the SIMT emulator.

What each case aims at:
  * seeds accepted and rejected, rewalks: ook_bursts (bursts across segment and warm-up starts);
  * successive rejections, >= 3 rounds: burst_over_many_segments;
  * a package open across a segment start, begun inside the warm-up (accepted) and in front of it (rejected), and
    every compared field group perturbed in such seeds: open_packages_at_segment_starts;
  * the FM state, the carried IQ sample and the FSK sub-detector in the comparison: fsk_fm_on (minmax, classic);
  * the load-time conversions: cs8_and_cf32; other detector levels and a wrapping FM filter: levels_and_low_pass;
  * hostile_families, ragged_mixed_batch, segment_sizes (1, 2, 3 blocks, warm-ups 1 and 2, SPLIT_AUTO);
  * every seed rejected (R433B_SPOIL_SEED), arena overflow (R433B_TEST_CAPS), submit / wait, the schedules that do
    not split, and the command line."""
import numpy as np
import pytest

import helpers
import hostile_iq as H
from oracle import refh
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OOK_RATE, FSK_RATE = 250000, 1024000
WRAPPING = 0.6  # FM low-pass above 0.5: a filter that is not provably monotone


def _pieces(make, seed, n, piece):
    """n samples of `make` (ook_stream / fsk_stream) in pieces of `piece` samples, each with as many bursts (<= 3) as
    fit in it (a piece too short for one is the start of a longer one)."""
    out, left, j = [], n, 0
    while left > 0:
        m = min(left, piece)
        for b in (3, 2, 1, -1):
            try:
                out.append(make(1000 * seed + j, m, b) if b >= 0 else make(1000 * seed + j, piece, 1)[:2 * m])
                break
            except ValueError:
                pass
        left -= m
        j += 1
    return np.concatenate(out)


def ook(seed, n):
    return _pieces(lambda s, m, b: synth.ook_stream(s, n_samples=m, n_bursts=b, kinds=("manchester", "silvercrest")),
                   seed, n, 1 << 16)


def fsk(seed, n):
    return _pieces(lambda s, m, b: synth.fsk_stream(s, n_samples=m, n_bursts=b), seed, n, 1 << 17)


def _pack(streams):
    """uint8 arrays -> (data, offsets, lengths), every stream start 32-byte aligned."""
    lens = [len(c) for c in streams]
    stride = [(n + 31) // 32 * 32 for n in lens]
    offsets = np.concatenate([[0], np.cumsum(stride)]).astype(np.uint64)
    data = np.zeros(max(int(offsets[-1]), 32), np.uint8)
    for c, o in zip(streams, offsets[:-1]):
        data[int(o):int(o) + len(c)] = c
    return data, offsets, lens


def run(ctx, streams, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=4096, split=0, warmup=1,
        analyze=False, grab=False, submit=False):
    """One batch of `streams` (uint8 arrays) -> what the comparison looks at, and the timing."""
    data, offsets, lens = _pack([s.view(np.uint8).ravel() for s in streams])
    ctx.set_split(split, warmup)
    try:
        if submit:
            ctx.submit(data, offsets, fmt, rate, freq, fpdm, block_bytes, lengths=lens)
            res = ctx.wait()
        else:
            ctx.process(data, offsets, fmt, rate, freq, fpdm, block_bytes, lengths=lens)
            res = ctx.fetch()
    finally:
        ctx.set_split(0)
    out = {"tm": ctx.timing(), "streams": [], "digests": []}
    for i in range(len(lens)):
        pk = res["packages"][res["packages"]["stream"] == i]
        hdr = [(int(k["seq"]), int(k["end_pos"])) for k in pk]
        out["streams"].append((helpers.gpu_stream_results(ctx, i), hdr))
        out["digests"].append(ctx.stream_digest(i))
    if analyze:
        ctx.analyze()
        out["text"] = [ctx.analysis(j)[2] for j in range(res["n_packages"])]
    if grab:
        plan = ctx.grab_plan(lib.GRAB_ALL)
        out["grab"] = (plan.tobytes(), ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes() if len(plan) else b"")
    return out


def same(got, want, tag):
    assert len(got["streams"]) == len(want["streams"])
    for i, ((g, gh), (w, wh)) in enumerate(zip(got["streams"], want["streams"])):
        d = helpers.compare_results(w, g, f"{tag} stream {i}", stages=False)
        assert not d, "\n".join(d[:20])
        assert gh == wh, f"{tag} stream {i}: (seq, end_pos) {gh[:8]} != {wh[:8]}"
    assert got["digests"] == want["digests"], tag
    for k in ("text", "grab"):
        if k in want:
            assert got[k] == want[k], f"{tag}: {k} differs"


def compare(ctx, streams, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=4096, split=2, warmup=1, tag="",
            **kw):
    """Split against unsplit in one context; returns the split run's timing."""
    want = run(ctx, streams, fmt, rate, freq, fpdm, block_bytes, **kw)
    assert want["tm"]["split_segments"] == 0
    assert any(s["packages"] for s, _ in want["streams"]), f"{tag}: no packages, nothing checked"
    got = run(ctx, streams, fmt, rate, freq, fpdm, block_bytes, split, warmup, **kw)
    same(got, want, tag)
    tm = got["tm"]
    assert tm["split_segments"] > len(streams), (tag, tm)
    assert tm["split_rewalks"] <= tm["split_segments"] - len(streams), (tag, tm)
    assert tm["detect_launches"] == 2 + tm["split_rounds"], (tag, tm)
    return tm, want


def vs_reference(want, streams, ss, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=4096, tag=""):
    """The unsplit run against the compiled reference, where it is present."""
    if not refh.available():
        return
    r = refh.Ref(store_bitbuffers=False, store_stages=False)
    r.register_defaults()
    for i, f in enumerate(streams):
        d = helpers.compare_results(r.run(f, ss, rate, freq, fpdm, block_bytes), want["streams"][i][0], f"{tag} {i} vs reference",
                                    stages=False)
        assert not d, "\n".join(d[:20])


# ------------------------------------------------------------------------------------------------------- cases ------

def ook_bursts(ctx, devices, n=1 << 18):
    """Bursts all over two cu8 streams of 2048-sample blocks, three blocks per segment: some land across segment starts
    and warm-up starts (seeds rejected, walked again), most segments start in noise (seeds accepted).  With the analyzer
    text and the -S all grab plan, and the unsplit run against the compiled reference."""
    streams = [ook(k, n) for k in (900, 901)]
    tm, want = compare(ctx, streams, lib.FMT_CU8, OOK_RATE, split=3, tag="ook", analyze=True, grab=True)
    assert 0 < tm["split_rewalks"] < tm["split_segments"] - len(streams), tm
    vs_reference(want, streams, 2, OOK_RATE, tag="ook")


def test_ook_bursts(ctx, devices):
    ook_bursts(ctx, devices)


def burst_over_many_segments(ctx, devices, n_pulses=600):
    """One pulse train that spans many one-block segments: each segment inside it starts inside a package whose start
    its warm-up cannot see, so successive seeds are rejected and the rewalks take one round per segment."""
    x = synth.ook_train_stream(905, n_pulses, n_samples=1 << 18)
    tm, _ = compare(ctx, [x], lib.FMT_CU8, OOK_RATE, split=1, tag="long burst")
    assert tm["split_rounds"] >= 3, tm


def test_burst_over_many_segments(ctx, devices):
    burst_over_many_segments(ctx, devices)


def trains_at(seed, starts, n_samples, n_pulses=30, period=100):
    """cu8 noise with one on/off keyed train of `n_pulses` pulses (period samples, half on) from each of `starts`."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(2 * n_samples, dtype=np.float32) * np.float32(2.0) + np.float32(127.5)
    on = ((np.arange(n_pulses * period) % period) < period // 2).astype(np.float32) * np.float32(80.0)
    for p in starts:
        ph = rng.uniform(0, 2 * np.pi) + 2 * np.pi * 0.05 * np.arange(len(on))
        x[2 * p:2 * (p + len(on)):2] += on * np.cos(ph).astype(np.float32)
        x[2 * p + 1:2 * (p + len(on)) + 1:2] += on * np.sin(ph).astype(np.float32)
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)


SEG, WARM, BLOCK_SAMPLES = 6, 2, 2048  # blocks per segment, warm-up blocks, cu8 samples of a 4096-byte block


def open_packages_at_segment_starts(ctx, devices, monkeypatch):
    """Every segment start lies inside a package.  Where the package began inside the warm-up, the seed equals the exact
    state with the package open (its trains included) and is accepted; where it began in front of the warm-up it is
    rejected.  Then R433B_SPOIL_SEED on the accepted seeds: every one is rejected, so no compared field group (the open
    package's trains, the carrier estimate, low, lead_in, ...) is left out of the comparison."""
    seg = SEG * BLOCK_SAMPLES
    n_segs = 12
    inside = trains_at(1100, [k * seg - 1500 for k in range(1, n_segs)], n_segs * seg)
    before = trains_at(1101, [k * seg - WARM * BLOCK_SAMPLES - 1500 for k in range(1, n_segs)], n_segs * seg, n_pulses=60)
    tm, _ = compare(ctx, [inside], lib.FMT_CU8, OOK_RATE, split=SEG, warmup=WARM, tag="open, begun in the warm-up")
    assert tm["split_segments"] == n_segs and tm["split_rewalks"] == 0, tm
    tm, _ = compare(ctx, [before], lib.FMT_CU8, OOK_RATE, split=SEG, warmup=WARM, tag="open, begun before it")
    assert tm["split_rewalks"] == n_segs - 1, tm
    monkeypatch.setenv("R433B_SPOIL_SEED", "1")
    c = lib.Context()
    try:
        c.set_devices(devices)
        tm, _ = compare(c, [inside], lib.FMT_CU8, OOK_RATE, split=SEG, warmup=WARM, tag="open, spoiled")
        assert tm["split_rewalks"] == n_segs - 1, tm
    finally:
        c.close()


def test_open_packages_at_segment_starts(ctx, devices, monkeypatch):
    open_packages_at_segment_starts(ctx, devices, monkeypatch)


def fsk_fm_on(ctx, devices, n=1 << 18):
    """cs16 2-FSK with FM on, minmax and classic: the FM filter state, the carried IQ sample and the FSK sub-detector
    are part of every comparison."""
    streams = [fsk(910 + k, n) for k in range(2)]
    for fpdm, freq in ((lib.FPDM_AUTO, 868000000), (lib.FPDM_CLASSIC, 433920000)):
        tm, want = compare(ctx, streams, lib.FMT_CS16, FSK_RATE, freq, fpdm, block_bytes=16384, split=2,
                           tag=f"fsk fpdm {fpdm}")
        assert any(p["type"] == 2 for s, _ in want["streams"] for p in s["packages"])
        assert tm["split_rewalks"] > 0, tm


def test_fsk_fm_on(ctx, devices):
    fsk_fm_on(ctx, devices)


def cs8_and_cf32(ctx, devices, n=1 << 17):
    cu8 = ook(915, n)
    cs8 = (cu8.astype(np.int16) - 128).astype(np.int8)
    compare(ctx, [cs8], lib.FMT_CS8, OOK_RATE, split=2, tag="cs8")
    cs16 = fsk(916, n)
    cf32 = (cs16.astype(np.float32) / np.float32(32768.0)).astype(np.float32)
    compare(ctx, [cf32], lib.FMT_CF32, FSK_RATE, 868000000, block_bytes=16384, split=2, tag="cf32")


def test_cs8_and_cf32(ctx, devices):
    cs8_and_cf32(ctx, devices)


def levels_and_low_pass(ctx, devices, n=1 << 17):
    """Magnitude mode at a non-default level point of tests/test_level_fuzz.py's grid, and a wrapping FM filter."""
    streams = [ook(920, n)]
    ctx.set_levels(1, -30.0, -12.1442, 9.0)
    try:
        compare(ctx, streams, lib.FMT_CU8, OOK_RATE, split=2, tag="magnitude, level -30")
    finally:
        ctx.set_levels()
    ctx.set_fm_low_pass(WRAPPING)
    try:
        compare(ctx, [fsk(921, n)], lib.FMT_CS16, FSK_RATE, 868000000,
                block_bytes=16384, split=2, tag="wrapping low-pass")
    finally:
        ctx.set_fm_low_pass(0.0)


def test_levels_and_low_pass(ctx, devices):
    levels_and_low_pass(ctx, devices)


def hostile_families(ctx, devices, seeds=(0, 1)):
    """Every hostile-IQ family of tests/hostile_iq.py, its cases concatenated into long streams (cu8 and cs16)."""
    cu8, cs16 = [], []
    for name, (make, _) in H.FAMILIES.items():
        for seed in seeds:
            for case in make(seed):
                (cs16 if case.fmt == lib.FMT_CS16 else cu8).append(case.iq.view(np.uint8).ravel())
    compare(ctx, [np.concatenate(cu8)], lib.FMT_CU8, H.RATE, split=2, tag="hostile cu8")
    if cs16:
        compare(ctx, [np.concatenate(cs16)], lib.FMT_CS16, FSK_RATE, 868000000, block_bytes=16384, split=2,
                tag="hostile cs16")


def test_hostile_families(ctx, devices):
    hostile_families(ctx, devices)


def ragged_mixed_batch(ctx, devices, n=1 << 17):
    """Split and unsplit streams of ragged lengths in one batch; the long ones end in a part of a block."""
    streams = [ook(930, n + 777), ook(931, 3000),
               ook(932, n // 2 + 1234), ook(933, 5000)]
    tm, _ = compare(ctx, streams, lib.FMT_CU8, OOK_RATE, split=3, tag="ragged")
    blocks = [-(-s.view(np.uint8).size // 4096) for s in streams]
    assert tm["split_segments"] == sum(-(-b // 3) for b in blocks), tm


def test_ragged_mixed_batch(ctx, devices):
    ragged_mixed_batch(ctx, devices)


def segment_sizes(ctx, devices, n=1 << 17):
    streams = [ook(940, n)]
    want = run(ctx, streams, lib.FMT_CU8, OOK_RATE)
    for seg, warm in ((1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (lib.SPLIT_AUTO, 1)):
        got = run(ctx, streams, lib.FMT_CU8, OOK_RATE, split=seg, warmup=warm)
        same(got, want, f"segment {seg} warm-up {warm}")
        assert got["tm"]["split_segments"] > 1, (seg, warm, got["tm"])
    with pytest.raises(lib.R433Error):
        ctx.set_split(2, 3)
    with pytest.raises(lib.R433Error):
        ctx.set_split(2, 0)


def test_segment_sizes(ctx, devices):
    segment_sizes(ctx, devices)


def test_more_slots_than_resident_warps(ctx, devices):
    """One-block segments of a 9 x 2^20-sample stream: 4608 slots, more than the 132 x 32 resident warps."""
    x = np.concatenate([ook(950 + k, 1 << 20) for k in range(9)])
    tm, _ = compare(ctx, [x], lib.FMT_CU8, OOK_RATE, split=1, tag="many slots")
    assert tm["split_segments"] > 132 * 32, tm


def spoiled_seeds(devices, monkeypatch, n=1 << 17):
    """R433B_SPOIL_SEED=1 perturbs every seed before the comparison: every seed is rejected, every segment but a
    stream's first is walked again, and the results do not change."""
    monkeypatch.setenv("R433B_SPOIL_SEED", "1")
    c = lib.Context()
    try:
        c.set_devices(devices)
        streams = [ook(960, n), fsk(961, n)]
        tm, _ = compare(c, streams[:1], lib.FMT_CU8, OOK_RATE, split=2, tag="spoiled ook")
        assert tm["split_rewalks"] == tm["split_segments"] - 1, tm
        tm, _ = compare(c, streams[1:], lib.FMT_CS16, FSK_RATE, 868000000, block_bytes=16384, split=1, tag="spoiled fsk")
        assert tm["split_rewalks"] == tm["split_segments"] - 1, tm
    finally:
        c.close()


def test_spoiled_seeds(devices, monkeypatch):
    spoiled_seeds(devices, monkeypatch)


def arena_overflow(devices, monkeypatch, n=1 << 17):
    """Package arenas far too small (R433B_TEST_CAPS): the split schedule grows them and runs again from pass 0."""
    streams = [ook(970, n)]
    c = lib.Context()
    try:
        c.set_devices(devices)
        want = run(c, streams, lib.FMT_CU8, OOK_RATE)
        ref = run(c, streams, lib.FMT_CU8, OOK_RATE, split=2)
    finally:
        c.close()
    monkeypatch.setenv("R433B_TEST_CAPS", "2,64,0")
    c = lib.Context()
    try:
        c.set_devices(devices)
        got = run(c, streams, lib.FMT_CU8, OOK_RATE, split=2)
    finally:
        c.close()
    same(got, want, "overflow")
    tm = got["tm"]
    assert tm["split_segments"] == ref["tm"]["split_segments"], tm
    assert tm["detect_launches"] > 2 + tm["split_rounds"], tm  # the attempts that overflowed count too


def test_arena_overflow(devices, monkeypatch):
    arena_overflow(devices, monkeypatch)


def submit_and_wait(ctx, devices, n=1 << 17):
    streams = [ook(980, n)]
    tm, _ = compare(ctx, streams, lib.FMT_CU8, OOK_RATE, split=2, tag="submit", submit=True)


def test_submit_and_wait(ctx, devices):
    submit_and_wait(ctx, devices)


def unsplit_schedules(ctx, devices, n=1 << 16):
    """Stage arrays, chained batches and batches without a stream of two segments run the existing schedules."""
    x = ook(990, n)
    data, offsets, lens = _pack([x])
    ctx.set_split(1)
    try:
        ctx.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=4096, lengths=lens, want_stages=True)
        assert ctx.timing()["split_segments"] == 0
        with lib.Chain(ctx, 1) as chain:
            ctx.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=4096, lengths=lens, chain=chain, last=[1])
            assert ctx.timing()["split_segments"] == 0
        short = x[:4096]
        d2, o2, l2 = _pack([short])
        ctx.process(d2, o2, lib.FMT_CU8, OOK_RATE, block_bytes=4096, lengths=l2)
        assert ctx.timing()["split_segments"] == 0
        ctx.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=4096, lengths=lens)
        assert ctx.timing()["split_segments"] > 1
    finally:
        ctx.set_split(0)


def test_unsplit_schedules(ctx, devices):
    unsplit_schedules(ctx, devices)


def command_line(capsys, tmp_path, n=1 << 19):
    """`python -m rtl_433_b200.captures FILES --split N|auto` prints what the plain run prints and grabs the same files
    with -S all; --split with --chunk-mb is refused."""
    from rtl_433_b200 import captures
    files = {"a_433.92M_250k.cu8": ook(995, n + 4321),
             "b_433.92M_250k.cu8": ook(996, 1 << 14),
             "f_868M_1024k.cs16": fsk(997, n)}
    paths = []
    for name, arr in files.items():
        arr.tofile(tmp_path / name)
        paths.append(str(tmp_path / name))
    outs = {}
    for tag, extra in (("plain", []), ("split", ["--split", "1"]), ("auto", ["--split"])):
        d = tmp_path / f"grab_{tag}"
        d.mkdir()
        captures.main(paths + extra + ["-S", "all", "--grab-dir", str(d)])
        outs[tag] = (capsys.readouterr().out, {p.name: p.read_bytes() for p in sorted(d.iterdir())})
    assert outs["plain"][0].count("package(s)") == 3 and outs["plain"][1]
    assert outs["split"] == outs["plain"]
    assert outs["auto"] == outs["plain"]
    with pytest.raises(SystemExit):
        captures.main(paths + ["--split", "2", "--chunk-mb", "1"])
    assert "--split does not run with --chunk-mb" in capsys.readouterr().err


def test_command_line(capsys, tmp_path):
    command_line(capsys, tmp_path)
