"""-m gpu: segmented replay on chained batches (include/r433b.h: r433b_chain_split).  Every case runs three ways: the
uncut files as one batch, the same chunks through a chain, and the same chunks through a chain that splits them.  All
three must be equal with nothing relaxed: every package field (seq and end_pos included), the pulse and gap widths,
every event of every (package, device) pair; the two chains also per batch in their stream digests and, where asked,
the analyzer text and the `-S all` grab plan with its bytes.  The uncut run is checked against the compiled reference
where it is present.  Each case asserts from r433b_timing that batches took the split path.
tests/test_emu_chain_split.py runs the same bodies, smaller, under the SIMT emulator.

What each case aims at:
  * segment 0 starting from a package the chain carried open across a chunk boundary, bursts across segment and
    warm-up starts: ook_bursts_across_boundaries;
  * the FM state, the carried IQ sample and the FSK sub-detector: fsk_minmax_and_classic; cs8_and_cf32;
  * ragged_slots (files ending in different rounds, empty chunks, a second file restarting seq);
  * chunk_and_segment_sizes; split_changed_mid_file; spoiled_seeds; arena_overflow; grabbing_chain;
    decoders_and_analyzer; argument_errors; set_split_does_not_split_chains."""
import numpy as np
import pytest

import test_chain as tc
import test_split as ts
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OOK_RATE, FSK_RATE = 250000, 1024000


def run_chain(ctx, slots, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, split=None, analyze=False,
              grab=False):
    """slots[i] = the files of slot i in order, each a list of chunks (as test_chain.run_chained).  split(r) -> the
    (segment_blocks, warmup_blocks) of round r's r433b_chain_split; None: the chain never opts in.
    -> ([[result per file] per slot], [per round: timing, digests and where asked analyzer text and grab plan])"""
    queues = [[(c, j == len(f) - 1, fi) for fi, f in enumerate(files) for j, c in enumerate(f)] for files in slots]
    out = [[tc._empty() for _ in files] for files in slots]
    rounds = []
    with lib.Chain(ctx, len(slots)) as chain:
        if grab:
            chain.grab(lib.GRAB_ALL)
        for r in range(max(len(q) for q in queues)):
            if split is not None:
                chain.split(*split(r))
            items = [q[r] if r < len(q) else (np.zeros(0, np.uint8), True, None) for q in queues]
            data, offsets, lens = tc._pack([c for c, _, _ in items])
            ctx.process(data, offsets, fmt, rate, freq, fpdm, block_bytes, lengths=lens, chain=chain,
                        last=[int(last) for _, last, _ in items])
            res = ctx.fetch()
            rd = {"tm": ctx.timing(), "digests": [ctx.stream_digest(i) for i in range(len(slots))]}
            for i, (c, _, fi) in enumerate(items):
                if fi is not None:
                    tc._add(out[i][fi], ctx, res, i, 0, False)
            if analyze:
                ctx.analyze()
                rd["text"] = [ctx.analysis(j)[2] for j in range(res["n_packages"])]
            if grab:
                plan = ctx.grab_plan(lib.GRAB_ALL)
                rd["grab"] = (plan.tobytes(),
                              ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes() if len(plan) else b"")
            rounds.append(rd)
    return [[tc._finish(a, False) for a in files] for files in out], rounds


def split_taken(rounds, n_slots, tag, overflow=False):
    """At least one batch took the split path; every batch that did ran pass 0, pass 1 and its rounds (plus, after
    an arena overflow, the attempts before)."""
    taken = [r["tm"] for r in rounds if r["tm"]["split_segments"]]
    assert any(tm["split_segments"] > n_slots for tm in taken), (tag, [r["tm"] for r in rounds])
    for tm in taken:
        assert tm["split_rewalks"] <= tm["split_segments"] - n_slots, (tag, tm)
        if not overflow:
            assert tm["detect_launches"] == 2 + tm["split_rounds"], (tag, tm)
    return taken


def three_ways(ctx, slots, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, split=lambda r: (2, 1),
               ref_ss=None, tag="", analyze=False, grab=False, split_ctx=None):
    """Uncut, chained and chained + split (in split_ctx when given); returns the split chain's rounds."""
    files = [np.concatenate(f) if f else np.zeros(0, np.uint8) for s in slots for f in s]
    want = tc.run_uncut(ctx, files, fmt, rate, freq, fpdm, block_bytes, stages=False)
    plain, plain_rounds = run_chain(ctx, slots, fmt, rate, freq, fpdm, block_bytes, None, analyze, grab)
    got, rounds = run_chain(split_ctx or ctx, slots, fmt, rate, freq, fpdm, block_bytes, split, analyze, grab)
    assert all(r["tm"]["split_segments"] == 0 for r in plain_rounds), tag
    assert any(w["packages"] for w in want), f"{tag}: no packages, nothing checked"
    j = 0
    for s, sl in enumerate(slots):
        for fi in range(len(sl)):
            tc.check(plain[s][fi], want[j], f"{tag} chained slot {s} file {fi}", stages=False)
            tc.check(got[s][fi], want[j], f"{tag} split slot {s} file {fi}", stages=False)
            j += 1
    assert len(rounds) == len(plain_rounds)
    for r, (g, w) in enumerate(zip(rounds, plain_rounds)):
        for k in ("digests", "text", "grab"):
            if k in w:
                assert g[k] == w[k], f"{tag} round {r}: {k} differs"
    if ref_ss:
        tc.vs_reference(want, files, ref_ss, rate, freq, fpdm, block_bytes, tag=tag)
    return rounds


def chunks(x, block, every):
    """x cut every `every` blocks (the last chunk ragged)."""
    n = x.view(np.uint8).size // block + 1
    return tc.cut(x, block, range(every, n, every))


# ------------------------------------------------------------------------------------------------------- cases ------

def ook_bursts_across_boundaries(ctx, devices, n=1 << 18):
    """cu8 in 4096-byte blocks, chunks of 16 blocks cut into segments of 3 behind 1- and 2-block warm-ups.  Slot 0
    holds pulse trains that begin in front of every chunk boundary (segment 0 of the next chunk starts inside the
    package the chain carried open) and in front of segment and warm-up starts; slot 1 holds bursts all over.  With
    the analyzer text, and the uncut run against the reference."""
    blk, chunk = 2048, 16 * 2048  # samples
    starts = [k * chunk - 1500 for k in range(1, n // chunk)]
    starts += [k * chunk + 3 * blk - 700 for k in range(n // chunk - 1)]         # across a segment start
    starts += [k * chunk + 6 * blk - 2 * blk - 900 for k in range(n // chunk - 1)]  # in front of a warm-up
    trains = ts.trains_at(1200, sorted(starts), n, n_pulses=25)
    slots = [[chunks(trains, 4096, 16)], [chunks(ts.ook(1201, n), 4096, 16)]]
    for warm in (1, 2):
        rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, split=lambda r: (3, warm),
                            ref_ss=2 if warm == 1 else None, tag=f"ook warm-up {warm}", analyze=True)
        taken = split_taken(rounds, 2, "ook")
        assert sum(tm["split_rewalks"] for tm in taken) > 0, taken


def test_ook_bursts_across_boundaries(ctx, devices):
    ook_bursts_across_boundaries(ctx, devices)


def fsk_minmax_and_classic(ctx, devices, n=1 << 18):
    """cs16 2-FSK with FM on in chunks of 4 blocks of 16 KiB, one-block segments: minmax and classic."""
    files = [ts.fsk(1210 + k, n) for k in range(2)]
    for fpdm, freq in ((lib.FPDM_AUTO, 868000000), (lib.FPDM_CLASSIC, 433920000)):
        rounds = three_ways(ctx, [[chunks(f, 16384, 4)] for f in files], lib.FMT_CS16, FSK_RATE, freq, fpdm, 16384,
                            split=lambda r: (1, 1), ref_ss=4, tag=f"fsk fpdm {fpdm}")
        split_taken(rounds, 2, f"fsk fpdm {fpdm}")


def test_fsk_minmax_and_classic(ctx, devices):
    fsk_minmax_and_classic(ctx, devices)


def cs8_and_cf32(ctx, devices, n=1 << 17):
    """cs8 (read as cu8) and cf32 (converted to cs16); cf32 chunks are whole multiples of 2 x block_bytes."""
    cs8 = (ts.ook(1220, n).astype(np.int16) - 128).astype(np.int8)
    split_taken(three_ways(ctx, [[chunks(cs8, 4096, 8)]], lib.FMT_CS8, OOK_RATE, block_bytes=4096, tag="cs8"), 1, "cs8")
    cf32 = (ts.fsk(1221, n).astype(np.float32) / np.float32(32768.0)).astype(np.float32)
    rounds = three_ways(ctx, [[chunks(cf32, 2 * 8192, 4)]], lib.FMT_CF32, FSK_RATE, 868000000, block_bytes=8192,
                        split=lambda r: (1, 1), tag="cf32")
    split_taken(rounds, 1, "cf32")


def test_cs8_and_cf32(ctx, devices):
    cs8_and_cf32(ctx, devices)


def ragged_slots(ctx, devices, n=1 << 17):
    """Files ending in different rounds and in a part of a block, an empty chunk that is not the last, an empty last
    chunk (flush only), and a slot that starts a second file (seq restarts at 0)."""
    blk = 4096
    empty = np.zeros(0, np.uint8)
    a = ts.ook(1230, n + 777)
    b = ts.ook(1231, n // 2)
    c = ts.ook(1232, n // 4 + 1234)
    d = ts.ook(1233, n // 2)
    ca = tc.cut(a, blk, [9, 10, 30])
    ca = ca[:2] + [empty] + ca[2:]
    slots = [[ca], [chunks(b, blk, 12) + [empty]], [chunks(c, blk, 7), chunks(d, blk, 10)]]
    rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=blk, ref_ss=2, tag="ragged")
    split_taken(rounds, 3, "ragged")


def test_ragged_slots(ctx, devices):
    ragged_slots(ctx, devices)


def chunk_and_segment_sizes(ctx, devices, n=1 << 17):
    """Chunks of 1, 3 and 16 blocks (1-block chunks never split), segments of 1-3 blocks with warm-ups 1 and 2, and
    SPLIT_AUTO."""
    x = ts.ook(1240, n)
    edges, k, sizes = [], 0, [1, 3, 16]
    while k * 4096 < x.size:
        k += sizes[len(edges) % 3]
        edges.append(k)
    slots = [[tc.cut(x, 4096, edges)]]
    for seg, warm in ((1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (lib.SPLIT_AUTO, 1)):
        rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, split=lambda r: (seg, warm),
                            tag=f"segment {seg} warm-up {warm}")
        split_taken(rounds, 1, f"segment {seg} warm-up {warm}")
        one_block = [r["tm"] for r, c in zip(rounds, slots[0][0]) if c.size <= 4096]
        assert one_block and all(tm["split_segments"] == 0 for tm in one_block), one_block


def test_chunk_and_segment_sizes(ctx, devices):
    chunk_and_segment_sizes(ctx, devices)


def split_changed_mid_file(ctx, devices, n=1 << 17):
    """r433b_chain_split turned on, off and changed between the chunks of open files."""
    plan = [(2, 1), (0, 1), (3, 2), (1, 1), (0, 1), (lib.SPLIT_AUTO, 1), (2, 2)]
    slots = [[chunks(ts.ook(1252 + k, n), 4096, 8)] for k in range(2)]
    rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, split=lambda r: plan[r % len(plan)],
                        tag="on / off")
    split_taken(rounds, 2, "on / off")
    for r, rd in enumerate(rounds):
        if plan[r % len(plan)][0] == 0:
            assert rd["tm"]["split_segments"] == 0, (r, rd["tm"])


def test_split_changed_mid_file(ctx, devices):
    split_changed_mid_file(ctx, devices)


def spoiled_seeds(ctx, devices, monkeypatch, n=1 << 17):
    """R433B_SPOIL_SEED=1: every seed is rejected, every segment but a chunk's first is walked again from its
    predecessor's end state (the first from the chain's), and the results do not change."""
    monkeypatch.setenv("R433B_SPOIL_SEED", "1")
    c = lib.Context()
    monkeypatch.delenv("R433B_SPOIL_SEED")
    try:
        c.set_devices(devices)
        slots = [[chunks(ts.ook(1260, n), 4096, 8)], [chunks(ts.ook(1261, n // 2), 4096, 8)]]
        rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, tag="spoiled", split_ctx=c)
        for tm in split_taken(rounds, 2, "spoiled"):
            assert tm["split_rewalks"] == tm["split_segments"] - 2, tm
    finally:
        c.close()


def test_spoiled_seeds(ctx, devices, monkeypatch):
    spoiled_seeds(ctx, devices, monkeypatch)


def arena_overflow(ctx, devices, monkeypatch, n=1 << 17):
    """Package arenas far too small (R433B_TEST_CAPS): the split schedule grows them and runs again from pass 0, from
    the state the chain carried; the next chunks' results are still equal (the chain state was not corrupted)."""
    monkeypatch.setenv("R433B_TEST_CAPS", "2,64,0")
    c = lib.Context()
    monkeypatch.delenv("R433B_TEST_CAPS")
    try:
        c.set_devices(devices)
        trains = ts.trains_at(1270, list(range(1000, n - 3000, 6000)), n, n_pulses=25)  # packages in every chunk
        slots = [[chunks(trains, 4096, 8)]]
        rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, tag="overflow", split_ctx=c)
        taken = split_taken(rounds, 1, "overflow", overflow=True)
        reran = [k for k, tm in enumerate(taken) if tm["detect_launches"] > 2 + tm["split_rounds"]]  # attempts count too
        assert reran and reran[0] + 1 < len(taken), taken  # an overflow, and a split batch behind it
    finally:
        c.close()


def test_arena_overflow(ctx, devices, monkeypatch):
    arena_overflow(ctx, devices, monkeypatch)


def grabbing_chain(ctx, devices, n=1 << 17):
    """r433b_chain_grab(-S all) on a splitting chain: every batch's plan and bytes equal the unsplit chain's."""
    slots = [[chunks(ts.ook(1280, n), 4096, 8)], [chunks(ts.ook(1281, n // 2), 4096, 5), chunks(ts.ook(1282, 9000), 4096, 2)]]
    rounds = three_ways(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, tag="grab", grab=True)
    split_taken(rounds, 2, "grab")
    assert any(r["grab"][0] for r in rounds), "no grabs, nothing checked"


def test_grabbing_chain(ctx, devices):
    grabbing_chain(ctx, devices)


def decoders_and_analyzer(devices, monkeypatch):
    """test_chain.decoders_and_analyzer's body with every chain split in one-block segments: the reference's decoders
    behind r433b_dispatch_r_devices, ungated and gated, give the uncut run's JSON, decode_* counters, sample_file_pos
    and analyzer text."""
    seen = []
    process = lib.Context.process

    class SplitChain(lib.Chain):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.split(1)

    def timed(self, *a, **kw):
        r = process(self, *a, **kw)
        if kw.get("chain") is not None:
            seen.append(self.timing())
        return r

    monkeypatch.setattr(lib, "Chain", SplitChain)
    monkeypatch.setattr(lib.Context, "process", timed)
    tc.decoders_and_analyzer(devices)
    assert any(tm["split_segments"] > 3 for tm in seen), seen


def test_decoders_and_analyzer(devices, monkeypatch):
    decoders_and_analyzer(devices, monkeypatch)


def argument_errors(ctx, devices):
    """warmup_blocks outside 1 .. segment_blocks, a null chain and a chain whose context is gone: R433B_EINVAL."""
    with lib.Chain(ctx, 1) as chain:
        for seg, warm in ((2, 3), (2, 0), (1, 2), (lib.SPLIT_AUTO, 0)):
            with pytest.raises(lib.R433Error, match="error -1"):
                chain.split(seg, warm)
        for seg, warm in ((0, 0), (0, 5), (2, 2), (lib.SPLIT_AUTO, 7)):
            chain.split(seg, warm)
    assert ctx.L.r433b_chain_split(None, 2, 1) == -1
    c = lib.Context()
    chain = lib.Chain(c, 1)
    c.L.r433b_destroy(c.h)  # the chain outlives its context
    c.h = None
    try:
        assert c.L.r433b_chain_split(chain.h, 2, 1) == -1
    finally:
        chain.close()
        c.close()


def test_argument_errors(ctx, devices):
    argument_errors(ctx, devices)


def set_split_does_not_split_chains(ctx, devices, n=1 << 17):
    """r433b_set_split is for unchained batches: a chain that did not opt in runs unsplit under it, with the same
    results; one that did splits whatever the context's setting."""
    slots = [[chunks(ts.ook(1290, n), 4096, 8)]]
    want, _ = run_chain(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096)
    ctx.set_split(1)
    try:
        got, rounds = run_chain(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096)
    finally:
        ctx.set_split(0)
    assert all(r["tm"]["split_segments"] == 0 for r in rounds), rounds
    tc.check(got[0][0], want[0][0], "set_split, no opt-in", stages=False)
    got, rounds = run_chain(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=4096, split=lambda r: (2, 1))
    split_taken(rounds, 1, "opt-in, set_split off")
    tc.check(got[0][0], want[0][0], "opt-in, set_split off", stages=False)


def test_set_split_does_not_split_chains(ctx, devices):
    set_split_does_not_split_chains(ctx, devices)
