"""Signal grabber on chained batches (include/r433b.h: r433b_chain_grab): every chain slot is its own grabber run.

For every slot, the grabs of a chained run equal those of one unchained batch that holds the slot's files in order
(tests/test_grab.py pins that path against the reference): the same list, grab_len, bytes, counter, run_end and every
window byte.  Each scenario also asserts that it reaches what it is there for, from the unchained plan's packages.
The bodies take the library as it is loaded, so tests/test_emu_chain_grab.py runs them under the SIMT emulator."""
import os
import tempfile

import numpy as np
import pytest

import test_grab as tg
from rtl_433_b200 import captures, lib, synth

RING = lib.GRAB_RING
RATE = synth.OOK_RATE


def _ss(fmt):
    return fmt & 0xff


def _in_div(fmt):
    return 2 if fmt == lib.FMT_CF32 else 1


def _records(ctx, mode, decoders, n_streams):
    """Plan and copy the fetched batch's grabs -> [dict] (window bytes as `data`), the plan."""
    if mode != lib.GRAB_ALL:
        decoders.dispatch(ctx, n_streams)
    if mode == lib.GRAB_UNDECODED:
        ctx.analyze()
    plan = ctx.grab_plan(mode)
    data = ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())) if len(plan) else np.zeros(0, np.uint8)
    out, at = [], 0
    for g in plan:
        n = int(g["bytes"])
        out.append({"stream": int(g["stream"]), "counter": int(g["counter"]), "grab_len": int(g["grab_len"]),
                    "bytes": n, "run_end": int(g["run_end"]), "data": data[at:at + n].tobytes()})
        at += n
    return out, plan


def _batch(chunks, fmt):
    """chunks (raw input bytes, one per stream) -> data, offsets, lengths: streams on a common stride."""
    align = 16 * _in_div(fmt)
    stride = max([align] + [(len(c) + align - 1) // align * align for c in chunks])
    data = np.zeros(stride * len(chunks), np.uint8)
    for i, c in enumerate(chunks):
        data[i * stride:i * stride + len(c)] = np.frombuffer(c, np.uint8)
    offsets = np.arange(len(chunks) + 1, dtype=np.uint64) * stride
    return data, offsets, np.array([len(c) for c in chunks], np.uint64)


def _process(ctx, data, offsets, lengths, fmt, rate, freq, block_bytes, on_device, **kw):
    keep = None
    if on_device:
        import torch
        keep = torch.from_numpy(data).cuda()
        data = keep.data_ptr()
    ctx.process(data, offsets, fmt, rate, freq, block_bytes=block_bytes, lengths=lengths, data_on_device=on_device, **kw)
    return keep


def unchained(ctx, files, fmt, mode, decoders=None, rate=RATE, freq=433920000, block_bytes=0):
    """One batch of `files` (one run) -> records, plan, packages, used bytes per file (after conversion)."""
    data, offsets, lengths = _batch(files, fmt)
    _process(ctx, data, offsets, lengths, fmt, rate, freq, block_bytes, False)
    res = ctx.fetch()
    recs, plan = _records(ctx, mode, decoders, len(files))
    used = [len(f) // 8 * 4 if fmt == lib.FMT_CF32 else len(f) for f in files]  # cf32 pairs -> cs16 bytes
    return recs, plan, res["packages"].copy(), used


def schedule(files, cadence, block_bytes, fmt, idle=(), empty_last=False):
    """A slot's calls: every file cut into chunks of `cadence` blocks, (raw bytes, last).  `idle`: call indices at which
    an empty chunk that is not the last goes in; empty_last: every file ends with an empty last chunk."""
    step = cadence * block_bytes * _in_div(fmt)
    calls = []
    for f in files:
        cut = [f[i:i + step] for i in range(0, len(f), step)] or [b""]
        if empty_last and len(cut[-1]) == step:
            cut.append(b"")
        calls += [(c, j == len(cut) - 1) for j, c in enumerate(cut)]
    for i in sorted(idle):
        calls.insert(i, (b"", False))
    return calls


def chained(ctx, slots, fmt, mode, decoders=None, rate=RATE, freq=433920000, block_bytes=0, on_device=False):
    """slots: per slot its calls (schedule()).  One chain, one batch per call -> per slot its records in call order,
    and every call's timing."""
    n = len(slots)
    n_calls = max(len(s) for s in slots)
    got = [[] for _ in range(n)]
    timings = []
    with lib.Chain(ctx, n) as ch:
        ch.grab(mode)
        for k in range(n_calls):
            calls = [s[k] if k < len(s) else (b"", False) for s in slots]
            data, offsets, lengths = _batch([c for c, _ in calls], fmt)
            keep = _process(ctx, data, offsets, lengths, fmt, rate, freq, block_bytes, on_device, chain=ch,
                            last=np.array([int(l) for _, l in calls], np.uint8))
            ctx.fetch()
            timings.append(ctx.timing())
            recs, _ = _records(ctx, mode, decoders, n)
            for r in recs:
                got[r.pop("stream")].append(r)
            del keep
    return got, timings


def reached(plan, pk, used, block_bytes, cadence, ss):
    """What the unchained run of one slot's files reaches -> set of names."""
    cum = np.concatenate([[0], np.cumsum(used)]).astype(np.int64)
    out = set()
    for g in plan:
        if not g["n_packages"]:
            continue
        p0, p1 = pk[g["first_package"]], pk[g["first_package"] + g["n_packages"] - 1]
        f = int(p1["stream"])
        n_blocks = -(-used[f] // block_bytes)
        b_first, b_last = int(p0["block"]), int(p1["block"])
        newest = cum[f] + min(used[f], (b_last + 2) * block_bytes)  # pushed after the call that ends the frame
        lo = int(g["run_end"]) - int(g["bytes"])
        if (b_last + 1) // cadence - b_first // cadence + 1 >= 3:
            out.add("spans 3 calls")
        if b_last + 1 >= n_blocks:
            out.add("ends at the flush")
        if lo < 0:
            out.add("before the run")
        if lo < newest - RING:
            out.add("newer bytes at wrapped slots")
        if f >= 1 and lo < cum[f]:
            out.add("reaches the previous file")
        if int(g["bytes"]) == RING and int(g["grab_len"]) * ss > RING:
            out.add("longer than the ring")
    return out


def compare(ctx, slot_files, slot_calls, fmt, mode, decoders=None, block_bytes=0, cadences=None, on_device=False,
            rate=RATE, freq=433920000, want=()):
    """Chained vs one unchained batch per slot; `want` names what the slots' runs must reach together."""
    got, timings = chained(ctx, slot_calls, fmt, mode, decoders, rate, freq, block_bytes, on_device)
    seen = set()
    for s, files in enumerate(slot_files):
        ref, plan, pk, used = unchained(ctx, files, fmt, mode, decoders, rate, freq, block_bytes)
        for r in ref:
            r.pop("stream")
        assert len(got[s]) == len(ref), (s, len(got[s]), len(ref))
        for i, (a, b) in enumerate(zip(got[s], ref)):
            assert a == b, (s, i, {k: (a[k], b[k]) for k in a if k != "data"}, a["data"] == b["data"])
        if cadences:
            seen |= reached(plan, pk, used, block_bytes or 262144, cadences[s], _ss(fmt))
    missing = set(want) - seen
    assert not missing, missing
    return got, timings


def _ook(seed, n, bursts, kinds=("silvercrest", "nice", "manchester"), decodable=False):
    return synth.ook_stream(seed, n_samples=n, n_bursts=bursts, kinds=kinds, decodable=decodable).tobytes()


def dense_ook(seed, seconds):
    """cu8 packed with 68 ms bursts 8 ms or more apart: frames run over many consecutive blocks."""
    n = int(seconds * RATE)
    return _ook(seed, n, int(0.95 * (n - 0.02 * RATE) / (0.076 * RATE)), ("nice", "manchester"))


def cadences_slots_and_files(ctx, mode=lib.GRAB_ALL, decoders=None, on_device=False, fmt=lib.FMT_CU8):
    """block_bytes 32768: three slots at 1, 2 and 4 blocks per call; a short first file closed by its flush whose
    window reaches before the run; frames over many calls; a second (and third) file per slot after `last`; empty
    chunks that are not the last, and empty last chunks."""
    bb = 32768
    conv = {lib.FMT_CU8: lambda b: b, lib.FMT_CS8: lambda b: tg._cs8(np.frombuffer(b, np.uint8)).tobytes()}[fmt]
    slot0 = [_ook(301, 60000, 1, ("nice",), True), dense_ook(302, 1.5)]
    slot1 = [_ook(311, 1 << 18, 6), _ook(312, 1 << 18, 6, ("silvercrest", "nice"), True), _ook(313, 40000, 0)]
    slot2 = [dense_ook(321, 1.2), _ook(322, 1 << 18, 5)]
    files = [[conv(f) for f in s] for s in (slot0, slot1, slot2)]
    calls = [schedule(files[0], 1, bb, fmt, idle=(3, 9)),
             schedule(files[1], 2, bb, fmt, empty_last=True),
             schedule(files[2], 4, bb, fmt, idle=(1,), empty_last=True)]
    assert any(len(c) == 0 and not l for c, l in calls[0]) and any(len(c) == 0 and l for c, l in calls[1])
    # what the frames reach is asserted on every frame (mode 1); modes 2-4 select among the same frames
    want = {"spans 3 calls", "ends at the flush", "before the run", "reaches the previous file"} if mode == lib.GRAB_ALL else ()
    return compare(ctx, files, calls, fmt, mode, decoders, block_bytes=bb, cadences=(1, 2, 4), on_device=on_device,
                   want=want)


def chunks_larger_than_the_ring(ctx):
    """Default blocks (256 KiB): 16 blocks per call is 4 MiB, more than the ring, so frames that end early in a chunk
    read the ring bytes its append overwrote; one slot at 1 block per call beside it.  Frames longer than the ring
    (clipped: "Signal bigger than buffer") read newer bytes at the ring's wrapped slots."""
    files = [[dense_ook(331, 9.0), _ook(332, 1 << 19, 6)], [_ook(333, 1 << 19, 5), dense_ook(334, 3.0)]]
    calls = [schedule(files[0], 16, 262144, lib.FMT_CU8), schedule(files[1], 1, 262144, lib.FMT_CU8)]
    compare(ctx, files, calls, lib.FMT_CU8, lib.GRAB_ALL, cadences=(16, 1),
            want={"longer than the ring", "newer bytes at wrapped slots", "reaches the previous file", "ends at the flush"})


def ring_appends(calls, fmt):
    """What k_grab_ring does for one slot's calls -> [(w0, n, shift, end)]: the ring position of the first appended
    byte, the bytes appended, the source's offset from 16-byte alignment there (chunks start 16-byte aligned) and the
    slot run's byte count after the append."""
    out, run = [], 0
    for c, _ in calls:
        used = len(c) // 8 * 4 if fmt == lib.FMT_CF32 else len(c)
        n = min(used, RING)
        w0 = (run + used - n) % RING
        run += used
        out.append((w0, n, (used - n - w0) % 16, run))
    return out


def _signal(fmt, seed, n, bursts):
    """n samples of OOK (cu8, cs8) or FSK (cs16) with up to `bursts` bursts -> raw bytes."""
    while True:
        try:
            if fmt == lib.FMT_CS16:
                return synth.fsk_stream(seed, n_samples=n, n_bursts=bursts).tobytes()
            x = synth.ook_stream(seed, n_samples=n, n_bursts=bursts, kinds=("silvercrest", "nice", "manchester"))
            return tg._cs8(x).tobytes() if fmt == lib.FMT_CS8 else x.tobytes()
        except ValueError:  # too many bursts for n samples
            bursts -= 1


def _dense_signal(fmt, seed, n, bursts):
    x = synth.ook_stream(seed, n_samples=n, n_bursts=bursts, kinds=("nice", "manchester"))
    return tg._cs8(x).tobytes() if fmt == lib.FMT_CS8 else x.tobytes()


def unaligned_ring_positions(ctx, fmt):
    """File lengths that are not multiples of 16 bytes, so the rings are written from positions that are not 16-byte
    aligned, through k_grab_ring's shifted words and its byte-wise ends: 3 blocks (of 32768 bytes) per call over a run
    past 3 MiB, and 100 blocks per call (more than the ring) after an unaligned first file, so that a whole ring is
    appended from an unaligned position."""
    bb = 32768
    ook = fmt != lib.FMT_CS16
    long = (1 << 21) + 7 if ook else (1 << 20) + 3
    # OOK: the long file is packed with bursts, so that frames run across the whole-ring append's end
    dense = int(0.95 * (long - 0.02 * RATE) / (0.076 * RATE)) if ook else 16
    files = [[_signal(fmt, 381, 60003, 1), _signal(fmt, 382, (1 << 18) + 5, 4), _signal(fmt, 383, 33333, 0),
              _signal(fmt, 384, 50001, 1), _signal(fmt, 385, (1 << 20) + 7, 12), _signal(fmt, 386, (1 << 18) + 1, 4)],
             [_signal(fmt, 391, 33333, 1), _dense_signal(fmt, 392, long, dense) if ook else _signal(fmt, 392, long, dense)]]
    calls = [schedule(files[0], 3, bb, fmt), schedule(files[1], 100, bb, fmt)]
    assert sum(len(f) for f in files[0]) > RING and any(len(f) % 16 for f in files[0] + files[1])
    appends = [ring_appends(c, fmt) for c in calls]
    every = appends[0] + appends[1]
    assert any(w0 % 16 and 0 < n < RING for w0, n, _, _ in every)   # partial words at both ends
    full = [end for w0, n, _, end in appends[1] if w0 % 16 and n == RING]
    assert full                                                       # a whole ring from an unaligned position
    assert any(shift and n >= 16 * 64 for _, n, shift, _ in every)   # shifted source words, the neighbour's by shuffle
    rate, freq = (synth.FSK_RATE, 868000000) if fmt == lib.FMT_CS16 else (RATE, 433920000)
    got, _ = compare(ctx, files, calls, fmt, lib.GRAB_ALL, block_bytes=bb, rate=rate, freq=freq)
    assert all(len(g) >= 1 for g in got), [len(g) for g in got]
    if ook:  # a window holds the last bytes of that append: the ones its first, shared ring word stores
        assert any(g["run_end"] - g["bytes"] <= end - 16 and end <= g["run_end"] for g in got[1] for end in full)


def fsk_formats(ctx):
    """cs16 and cf32 (grabbed as the cs16 it was converted to), 1 and 2 blocks per call."""
    x = [synth.fsk_stream(341 + i, n_samples=1 << 18, n_bursts=3) for i in range(3)]
    for fmt, files in ((lib.FMT_CS16, [v.tobytes() for v in x]), (lib.FMT_CF32, [tg._cf32(v).tobytes() for v in x])):
        slots = [files[:2], files[2:]]
        calls = [schedule(slots[0], 1, 262144, fmt), schedule(slots[1], 2, 262144, fmt)]
        got, _ = compare(ctx, slots, calls, fmt, lib.GRAB_ALL, rate=synth.FSK_RATE, freq=868000000)
        assert sum(len(g) for g in got) >= 3


def pipelined_host_input(ctx):
    """Host input through the time-sliced path (4 slices per call)."""
    ctx.set_pipeline(4)
    try:
        files = [[_ook(351, 1 << 18, 6), _ook(352, 1 << 18, 6)], [_ook(353, 1 << 19, 10)]]
        calls = [schedule(files[0], 2, 32768, lib.FMT_CU8), schedule(files[1], 2, 32768, lib.FMT_CU8)]
        _, timings = compare(ctx, files, calls, lib.FMT_CU8, lib.GRAB_ALL, block_bytes=32768)
        assert max(t["detect_launches"] for t in timings) > 1
    finally:
        ctx.set_pipeline(0)


def arena_overflow_rerun(devices, monkeypatch):
    """A context with small result arenas runs chained batches again (R433B_TEST_CAPS); the rings are appended once."""
    files = [[_ook(361, 1 << 18, 8), _ook(362, 1 << 18, 8)], [_ook(363, 1 << 19, 12)]]
    calls = [schedule(files[0], 2, 32768, lib.FMT_CU8), schedule(files[1], 4, 32768, lib.FMT_CU8)]
    monkeypatch.setenv("R433B_TEST_CAPS", "2,64,0")
    c = lib.Context(0)
    monkeypatch.delenv("R433B_TEST_CAPS")
    try:
        c.set_devices(devices)
        got, timings = chained(c, calls, lib.FMT_CU8, lib.GRAB_ALL, block_bytes=32768)
    finally:
        c.close()
    assert max(t["detect_launches"] for t in timings) > 1
    ref = lib.Context(0)
    try:
        ref.set_devices(devices)
        for s, f in enumerate(files):
            want, _, _, _ = unchained(ref, f, lib.FMT_CU8, lib.GRAB_ALL, block_bytes=32768)
            for r in want:
                r.pop("stream")
            assert got[s] == want, s
    finally:
        ref.close()


def golden_cases_one_slot(mode_cases=(("all", None),)):
    """tests/golden/grab.json replayed through one-slot chains (1 block per call): the reference's files."""
    ctx = lib.Context(0)
    try:
        with tempfile.TemporaryDirectory() as d:
            for case, modes in mode_cases:
                sub = os.path.join(d, case)
                os.makedirs(sub)
                paths = tg.write_case(tg.cases()[case], sub)
                bs = [captures.load_batches([p])[0] for p in paths]
                fmt, rate, freq = bs[0]["abi_format"], bs[0]["sample_rate"], bs[0]["center_frequency"]
                raw = [b["data"][int(b["offsets"][0]):int(b["offsets"][0]) + int(b["lengths"][0])].tobytes() for b in bs]
                for mode in modes:
                    decoders = tg.Decoders() if mode != "all" else None
                    try:
                        ctx.set_devices(decoders.devices if decoders else lib.default_device_table())
                        ctx.set_gates(None)
                        got, _ = chained(ctx, [schedule(raw, 1, 262144, fmt)], fmt, tg.MODES[mode], decoders, rate, freq)
                    finally:
                        if decoders:
                            decoders.close()
                    files = {captures.grab_name(g["counter"], freq, rate, _ss(fmt)): g["data"] for g in got[0]}
                    assert tg.fingerprint(files) == tg.golden()[case][mode], (case, mode)
    finally:
        ctx.close()


def state_errors(devices):
    """R433B_ESTATE: a plan on a chain that does not grab, grabbing enabled while a file is open, a chained batch after
    one that was not planned, r433b_grab_tail on a chained batch.  R433B_EINVAL: a prior, another mode."""
    x = np.frombuffer(_ook(371, 1 << 17, 2), np.uint8)
    block = 32768
    first = x[:4 * block]
    ctx = lib.Context(0)
    try:
        ctx.set_devices(devices)
        off = np.array([0, first.nbytes], np.uint64)
        with lib.Chain(ctx, 1) as ch:
            ctx.process(first, off, lib.FMT_CU8, RATE, 433920000, block_bytes=block, chain=ch, last=[0])
            ctx.fetch()
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ctx.grab_plan(lib.GRAB_ALL)
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ctx.grab_tail()
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ch.grab(lib.GRAB_ALL)
        with lib.Chain(ctx, 1) as ch:
            with pytest.raises(lib.R433Error, match="r433b error -1"):
                ch.grab(5)
            ch.grab(lib.GRAB_ALL)
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ch.grab(lib.GRAB_ALL)
            ctx.process(first, off, lib.FMT_CU8, RATE, 433920000, block_bytes=block, chain=ch, last=[0])
            ctx.fetch()
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ctx.process(first, off, lib.FMT_CU8, RATE, 433920000, block_bytes=block, chain=ch, last=[0])
            with pytest.raises(lib.R433Error, match="r433b error -1"):
                ctx.grab_plan(lib.GRAB_ALL, (0, np.zeros(0, np.uint8), 1))
            with pytest.raises(lib.R433Error, match="r433b error -1"):
                ctx.grab_plan(lib.GRAB_KNOWN)
            ctx.grab_plan(lib.GRAB_ALL)
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ctx.grab_tail()
            ctx.grab_plan(lib.GRAB_ALL)  # planning again is the same plan
            ctx.process(first, off, lib.FMT_CU8, RATE, 433920000, block_bytes=block, chain=ch, last=[1])
            ctx.fetch()
            ctx.grab_plan(lib.GRAB_ALL)
    finally:
        ctx.close()


@pytest.fixture(scope="module")
def devices():
    return lib.default_device_table()


@pytest.fixture(scope="module")
def ctx(devices):
    c = lib.Context(0)
    c.set_devices(devices)
    yield c
    c.close()


@pytest.mark.gpu
def test_cadences_slots_and_files(ctx):
    cadences_slots_and_files(ctx)


@pytest.mark.gpu
def test_device_input_and_cs8(ctx):
    if not lib.LIB_PATH.endswith("libr433b.so"):
        pytest.skip("device input needs device memory")
    cadences_slots_and_files(ctx, on_device=True)
    cadences_slots_and_files(ctx, fmt=lib.FMT_CS8)


@pytest.mark.gpu
def test_chunks_larger_than_the_ring(ctx):
    chunks_larger_than_the_ring(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [lib.FMT_CU8, lib.FMT_CS8, lib.FMT_CS16], ids=["cu8", "cs8", "cs16"])
def test_unaligned_ring_positions(ctx, fmt):
    unaligned_ring_positions(ctx, fmt)


@pytest.mark.gpu
def test_cs16_and_cf32(ctx):
    fsk_formats(ctx)


@pytest.mark.gpu
def test_pipelined_host_input(ctx):
    pipelined_host_input(ctx)


@pytest.mark.gpu
def test_arena_overflow_rerun(devices, monkeypatch):
    arena_overflow_rerun(devices, monkeypatch)


@pytest.mark.gpu
@tg.needs_ref
@pytest.mark.parametrize("mode", ["unknown", "known", "undecoded"])
def test_modes_with_reference_decoders(mode):
    decoders = tg.Decoders()
    c = lib.Context(0)
    try:
        c.set_devices(decoders.devices)
        cadences_slots_and_files(c, tg.MODES[mode], decoders)
    finally:
        c.close()
        decoders.close()


@pytest.mark.gpu
def test_golden_cases_one_slot():
    golden_cases_one_slot((("ook_cu8", ("all",)), ("ook_cs8", ("all",)), ("fsk_cs16", ("all",)), ("fsk_cf32", ("all",))))


@pytest.mark.gpu
@tg.needs_ref
def test_golden_modes_one_slot():
    golden_cases_one_slot((("ook_cu8", ("unknown", "known", "undecoded")),))


@pytest.mark.gpu
def test_state_errors(devices):
    state_errors(devices)
