"""-m gpu: mixed batches on chains (include/r433b.h: r433b_process_mixed_chained).  Slots of one chain carry files of
different sample formats, rates and centre frequencies, chunk by chunk.  For every slot, the merged results of the
chained calls must equal those of its files processed uncut and alone through r433b_process(), and those of one
unchained r433b_process_mixed() of the uncut files, with nothing relaxed: every r433b_package field but the ones that
say where it lies (seq, offset, end_pos and block included), the pulse and gap widths, every pair's counts and every
event, every pulse_data_t field and sample_file_pos, and the analyzer's text and trial events.
tests/test_emu_mixed_chain.py runs the same bodies, smaller, under the SIMT emulator."""
import ctypes as C

import numpy as np
import pytest

import test_chain as tc
import test_chain_grab as tcg
import test_grab as tg
import test_mixed as tm
from oracle import refh
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BLOCK = tm.BLOCK
EMPTY = np.zeros(0, np.uint8)
EINVAL, ESTATE = -1, -5  # R433B_EINVAL, R433B_ESTATE


def _in_div(fmt):
    return 2 if fmt == lib.FMT_CF32 else 1


def _raw(x):
    return x.view(np.uint8).ravel()


def calls_of(files, blocks, block_bytes=BLOCK, idle=(), empty_last=False):
    """A slot's calls: every file (tag, x, fmt, rate, freq) cut into chunks of `blocks` blocks of its own input ->
    [(file index or None, chunk bytes, last)].  idle: call indices at which an empty chunk that is not the last goes in
    (inside the file open there); empty_last: every file whose last chunk is whole ends with an empty last chunk."""
    calls = []
    for fi, (_, x, fmt, *_) in enumerate(files):
        b = _raw(x)
        step = blocks * block_bytes * _in_div(fmt)
        cut = [b[i:i + step] for i in range(0, len(b), step)] or [EMPTY]
        if empty_last and len(cut[-1]) == step:
            cut.append(EMPTY)
        calls += [(fi, c, j == len(cut) - 1) for j, c in enumerate(cut)]
    for i in sorted(idle):
        fi, _, last = calls[i - 1]
        assert not last, "an idle chunk goes inside a file"
        calls.insert(i, (fi, EMPTY, False))
    return calls


def class_order(fmts, rates, freqs, on_device=False):
    """The library's internal order (DESIGN §7d): streams sorted by class, stable in slot order -> slot per position."""
    def key(i):
        f = fmts[i]
        return (rates[i], f & 0xff, f == lib.FMT_CS8, freqs[i] > 800000000, f == lib.FMT_CF32 and on_device)
    return sorted(range(len(fmts)), key=key)


def _merge(acc, snap):
    if acc is None:
        snap = dict(snap)
        snap.pop("digest")
        return snap
    k0 = len(acc["results"]["packages"])
    acc["results"]["packages"] += snap["results"]["packages"]
    for e in snap["results"]["events"]:
        e["package"] += k0
        acc["results"]["events"].append(e)
    for k in ("headers", "pairs", "pulse_data", "analysis"):
        if k in acc:
            acc[k] += snap[k]
    return acc


def run_chain(ctx, slots, slot_calls, fpdm=lib.FPDM_AUTO, analyze=False, on_device=False, reverse=False,
              block_bytes=BLOCK, chain_setup=None, per_call=None):
    """slots[s]: slot s's files; slot_calls[s]: its calls (calls_of).  One mixed chained batch per round; a slot
    without a call gets an empty last chunk in the format of its last file (a new empty file, not collected).
    -> (per slot, per file: merged snapshot), [timing per call], [per call: (slot order, open before, seqs per slot)]."""
    n = len(slots)
    acc = [[None] * len(files) for files in slots]
    timings, log = [], []
    open_ = [False] * n
    with lib.Chain(ctx, n) as ch:
        if chain_setup:
            chain_setup(ch)
        for r in range(max(len(c) for c in slot_calls)):
            items, lasts, which = [], [], []
            for s in range(n):
                if r < len(slot_calls[s]):
                    fi, chunk, last = slot_calls[s][r]
                else:
                    fi, chunk, last = None, EMPTY, True
                _, _, fmt, rate, freq = slots[s][fi if fi is not None else -1]
                items.append(("", chunk, fmt, rate, freq))
                lasts.append(int(last))
                which.append(fi)
            data, offsets, lens = tm._pack(items, reverse)
            keep = None
            if on_device:
                import torch
                keep = torch.from_numpy(data).cuda()
                data = keep.data_ptr()
            fmts, rates, freqs = [t[2] for t in items], [t[3] for t in items], [t[4] for t in items]
            ctx.process_mixed(data, offsets, fmts, rates, freqs, lengths=lens, fpdm_mode=fpdm, data_on_device=on_device,
                              block_bytes=block_bytes, chain=ch, last=lasts)
            res = ctx.fetch()
            if analyze:
                ctx.analyze()
            timings.append(ctx.timing())
            pk = res["packages"]
            log.append((class_order(fmts, rates, freqs, on_device), list(open_),
                        [[int(k["seq"]) for k in pk[pk["stream"] == s]] for s in range(n)]))
            for s in range(n):
                if which[s] is not None:
                    acc[s][which[s]] = _merge(acc[s][which[s]], tm._drop_positions(tm.snapshot(ctx, res, s, analyze)))
            if per_call:
                per_call(ctx, res, ch)
            open_ = [not l for l in lasts]
            del keep
    return acc, timings, log


def expect(ctx, slots, fpdm=lib.FPDM_AUTO, analyze=False):
    """Every slot's files uncut and alone (r433b_process), and in one unchained mixed batch -> two [[snapshot]]."""
    flat = [f for files in slots for f in files]
    alone = tm.alone(ctx, flat, fpdm, analyze)
    mixed, _ = tm.mixed(ctx, flat, fpdm, analyze)
    out_a, out_m, k = [], [], 0
    for files in slots:
        out_a.append(alone[k:k + len(files)])
        out_m.append(mixed[k:k + len(files)])
        k += len(files)
    return out_a, out_m


def same(got, want, slots, tag):
    for s, files in enumerate(slots):
        for fi, f in enumerate(files):
            g, w = got[s][fi], dict(want[s][fi])
            w.pop("digest", None)
            t = f"{tag} slot {s} file {fi} ({f[0]})"
            assert g is not None, t + ": never processed"
            d = tc.helpers.compare_results(w["results"], g["results"], t, stages=False)
            assert not d, "\n".join(d[:20])
            for k in w:
                if k != "results":
                    assert g[k] == w[k], f"{t}: {k} differs"


def check(ctx, slots, slot_calls, fpdm=lib.FPDM_AUTO, analyze=False, tag="", **kw):
    want_alone, want_mixed = expect(ctx, slots, fpdm, analyze)
    assert sum(len(w["headers"]) for ws in want_alone for w in ws) > 3, "nothing detected: nothing checked"
    got, timings, log = run_chain(ctx, slots, slot_calls, fpdm, analyze, **kw)
    same(got, want_alone, slots, tag + " vs alone")
    same(got, want_mixed, slots, tag + " vs one mixed batch")
    assert all(t["split_segments"] == 0 for t in timings)
    return got, timings, log, want_alone


def spans_calls(log):
    """Whether some call continued a file whose earlier packages came in an earlier call (seq does not start at 0)."""
    return any(o and seqs and seqs[0] > 0 for _, open_, per in log for o, seqs in zip(open_, per))


# ---- parity over the corpus of test_mixed, one file per slot ------------------------------------------------------------

def corpus_parity(ctx, devices, n=1 << 17, blocks=3, on_device=False, gates=False, fpdm=lib.FPDM_AUTO, analyze=True,
                  reverse=False):
    slots = [[f] for f in tm.corpus(n)]
    ctx.set_gates(lib.default_gates(devices) if gates else None)
    try:
        _, timings, log, want = check(ctx, slots, [calls_of(s, blocks) for s in slots], fpdm, analyze,
                                      f"corpus blocks={blocks} device={on_device} gates={gates} fpdm={fpdm}",
                                      on_device=on_device, reverse=reverse)
    finally:
        ctx.set_gates(None)
    assert any(h[1] == lib.PACKAGE_FSK for ws in want for w in ws for h in w["headers"]), "no FSK package"
    if blocks < 16:
        assert spans_calls(log), "no file's packages came in more than one call"
    assert timings[0]["mixed_classes"] == 5, timings[0]
    return timings


# ---- slots that change format at file starts, so that the internal order changes from call to call ---------------------

def changing_slots(n=1 << 16):
    """Slot 0: cu8 250k, cs16 1024k FSK, cf32; slot 1: cs8 250k, cu8 2048k; slot 2: cs16 1024k, cu8 250k (short)."""
    ook = lambda seed, m, rate=250000: tm._ook(seed, m, rate)  # noqa: E731
    fsk = lambda seed, m: synth.fsk_stream(seed, n_samples=max(m, 1 << 16), n_bursts=1, rate=1024000)  # noqa: E731
    cf32 = (fsk(16, n).astype(np.float32) / np.float32(32767.0)).astype(np.float32)
    return [
        [("s0 cu8_250k", ook(11, n), lib.FMT_CU8, 250000, 433920000),
         ("s0 cs16_1024k", fsk(12, n), lib.FMT_CS16, 1024000, 868000000),
         ("s0 cf32_1024k", cf32, lib.FMT_CF32, 1024000, 868000000)],
        [("s1 cs8_250k", ook(13, n - 2000) ^ 0x80, lib.FMT_CS8, 250000, 315000000),
         ("s1 cu8_2048k", ook(14, n, 2048000), lib.FMT_CU8, 2048000, 433920000)],
        [("s2 cs16_1024k", fsk(15, n // 2), lib.FMT_CS16, 1024000, 915000000),
         ("s2 cu8_250k", ook(17, n // 2 + 1000), lib.FMT_CU8, 250000, 433920000)],
    ]


def order_changes(ctx, devices, n=1 << 16, on_device=False):
    slots = changing_slots(n)
    slot_calls = [calls_of(slots[0], 2, idle=(3,)), calls_of(slots[1], 3, empty_last=True),
                  calls_of(slots[2], 1, idle=(2, 5))]
    _, _, log, want = check(ctx, slots, slot_calls, analyze=False, tag="order changes", on_device=on_device)
    # a continuing slot changed its internal position, and seq went on across calls and restarted with each new file
    moved = any(o and a.index(s) != b.index(s)
                for (a, _, _), (b, open_, _) in zip(log, log[1:]) for s, o in enumerate(open_))
    assert moved, "no continuing slot changed its internal position"
    assert spans_calls(log), "no file's packages came in more than one call"
    restarted = [s for s in range(len(slots)) for fi in range(1, len(slots[s])) if want[s][fi]["headers"]
                 and want[s][fi - 1]["headers"]]
    assert restarted, "no slot began a file with packages after one with packages"


# ---- carried state in every class -------------------------------------------------------------------------------------

def carried_state_slots(n=1 << 16):
    m = max(n, 1 << 17)  # two FSK bursts at 1024k
    fsk = synth.fsk_stream(21, n_samples=m, n_bursts=2, rate=1024000)
    return [
        [("long ook", synth.ook_train_stream(20, n_pulses=300, n_samples=n), lib.FMT_CU8, 250000, 433920000)],
        [("fsk minmax", fsk, lib.FMT_CS16, 1024000, 868000000)],
        [("fsk classic", synth.fsk_stream(22, n_samples=m, n_bursts=2, rate=1024000), lib.FMT_CS16, 1024000, 433920000)],
        [("cs8", (synth.ook_stream(23, n_samples=n, n_bursts=2).astype(np.int16) - 128).astype(np.int8), lib.FMT_CS8,
          250000, 433920000)],
        [("cf32", (fsk.astype(np.float32) / np.float32(32767.0)).astype(np.float32), lib.FMT_CF32, 1024000, 868000000)],
    ]


def carried_state(ctx, devices, n=1 << 16, blocks=1):
    slots = carried_state_slots(n)
    _, timings, log, want = check(ctx, slots, [calls_of(s, blocks) for s in slots], tag="carried state")
    assert spans_calls(log)
    assert sum(t["chain_folds"] for t in timings) > 0
    assert sum(t["chain_fm_rebuilds"] for t in timings) > 0
    assert any(h[1] == lib.PACKAGE_FSK for ws in want for w in ws for h in w["headers"])


def spoiled_front(devices, monkeypatch, n=1 << 16):
    """R433B_SPOIL_FRONT=4 spoils tile 0 of every continued chunk: k_detect must find and repair it in every class."""
    slots = carried_state_slots(n)
    slot_calls = [calls_of(s, 1) for s in slots]
    monkeypatch.setenv("R433B_SPOIL_FRONT", "4")
    c = lib.Context(0)
    monkeypatch.delenv("R433B_SPOIL_FRONT")
    try:
        c.set_devices(devices)
        _, timings, log, _ = check(c, slots, slot_calls, tag="spoiled")
        for s, calls in enumerate(slot_calls):  # per class: one slot each, so one run per slot
            continued = sum(1 for k, (_, chunk, _) in enumerate(calls) if k and len(chunk))
            assert continued > 0
        continued = sum(1 for _, open_, _ in log for o in open_ if o)
        assert sum(t["front_repairs"] for t in timings) >= continued, (timings, continued)
    finally:
        c.close()


def arena_overflow(devices, monkeypatch, n=1 << 16):
    """Arenas far too small on calls whose packages are open across both boundaries: each reruns from the carried
    state, and every later call stays equal."""
    slots = carried_state_slots(n)[:3]
    c = lib.Context(0)
    c.set_devices(devices)
    want_alone, want_mixed = expect(c, slots)
    c.close()
    monkeypatch.setenv("R433B_TEST_CAPS", "4,64,256")
    c = lib.Context(0)
    try:
        c.set_devices(devices)
        got, _, log = run_chain(c, slots, [calls_of(s, 1) for s in slots])
        same(got, want_alone, slots, "overflow vs alone")
        same(got, want_mixed, slots, "overflow vs one mixed batch")
        assert spans_calls(log)
    finally:
        c.close()


# ---- equivalences -----------------------------------------------------------------------------------------------------

def one_format_equals_chained(ctx, devices, n=1 << 17, block_bytes=BLOCK):
    """A one-format mixed chain equals r433b_process_chained on the same chunks: packages, digests and grabs."""
    files = [("a", tm._ook(31, n, 250000), lib.FMT_CU8, 250000, 433920000), ("b", tm._ook(32, n - 1000, 250000), lib.FMT_CU8, 250000, 433920000)]
    slot_calls = [calls_of([f], k, block_bytes) for f, k in zip(files, (1, 3))]
    rounds = max(len(c) for c in slot_calls)
    runs = []
    for mixed in (False, True):
        out = []
        with lib.Chain(ctx, len(files)) as ch:
            ch.grab(lib.GRAB_ALL)
            for r in range(rounds):
                calls = [c[r] if r < len(c) else (None, EMPTY, True) for c in slot_calls]
                data, offsets, lens = tm._pack([("", c, *files[0][2:]) for _, c, _ in calls])
                last = [int(l) for _, _, l in calls]
                if mixed:
                    ctx.process_mixed(data, offsets, [lib.FMT_CU8] * 2, [250000] * 2, [433920000] * 2, lengths=lens,
                                      block_bytes=block_bytes, chain=ch, last=last)
                else:
                    ctx.process(data, offsets, lib.FMT_CU8, 250000, 433920000, block_bytes=block_bytes, lengths=lens,
                                chain=ch, last=last)
                res = ctx.fetch()
                recs, _ = tcg._records(ctx, lib.GRAB_ALL, None, len(files))
                pk = res["packages"].copy()
                pk["pulse_off"] = 0
                pk["first_pair"] = 0
                out.append((pk.tobytes(), [ctx.stream_digest(s) for s in range(len(files))], recs,
                            [ch.base(s) for s in range(len(files))]))
        runs.append(out)
    assert sum(len(np.frombuffer(o[0], lib.PACKAGE_DTYPE)) for o in runs[0]) >= 2
    for r, (a, b) in enumerate(zip(*runs)):
        assert a == b, f"call {r} differs"


def split_chain_unsplit(ctx, devices, n=1 << 16):
    """A chain that opted into r433b_chain_split runs a mixed batch unsplit, with equal results."""
    slots = changing_slots(n)
    slot_calls = [calls_of(s, 2) for s in slots]
    check(ctx, slots, slot_calls, tag="split chain", chain_setup=lambda ch: ch.split(1, 1))


# ---- the signal grabber ------------------------------------------------------------------------------------------------

def grab_slots(n):
    """Per slot its grab files (tag, x, fmt, rate, freq): cu8 (decodable) next to cs8 in the same calls, then cf32 and
    cs16."""
    def ook(seed, m, bursts, decodable=False):
        return synth.ook_stream(seed, n_samples=m, n_bursts=bursts, kinds=("silvercrest", "nexus"), decodable=decodable)
    fsk = synth.fsk_stream(410, n_samples=n // 2, n_bursts=2, rate=1024000)
    return [
        [("g0 cu8", ook(401, n, 3, decodable=True), lib.FMT_CU8, 250000, 433920000),
         ("g0 cs16", synth.fsk_stream(411, n_samples=n // 2, n_bursts=2, rate=1024000), lib.FMT_CS16, 1024000, 868000000)],
        [("g1 cs8", tg._cs8(ook(402, n, 3)), lib.FMT_CS8, 250000, 315000000),
         ("g1 cu8", ook(403, n // 2, 1), lib.FMT_CU8, 250000, 433920000)],
        [("g2 cf32", tg._cf32(fsk), lib.FMT_CF32, 1024000, 868000000)],
    ]


def grab_records_mixed(ctx, files, mode, decoders):
    """One unchained mixed batch of a slot's files in order -> grab records."""
    data, offsets, lens = tm._pack(files)
    ctx.process_mixed(data, offsets, [f[2] for f in files], [f[3] for f in files], [f[4] for f in files], lengths=lens)
    ctx.fetch()
    recs, _ = tcg._records(ctx, mode, decoders, len(files))
    for r in recs:
        r.pop("stream")
    return recs


def grabbing_chain(ctx, n=1 << 20, blocks=(1, 3), mode=lib.GRAB_ALL, decoders=None, on_device=False):
    slots = grab_slots(n)
    got = [[] for _ in slots]

    def per_call(c, res, ch):
        recs, _ = tcg._records(c, mode, decoders, len(slots))
        for r in recs:
            got[r.pop("stream")].append(r)

    slot_calls = [calls_of(s, blocks[i % len(blocks)], 262144) for i, s in enumerate(slots)]
    run_chain(ctx, slots, slot_calls, block_bytes=262144, on_device=on_device, chain_setup=lambda ch: ch.grab(mode),
              per_call=per_call)
    total = 0
    for s, files in enumerate(slots):
        want = grab_records_mixed(ctx, files, mode, decoders)
        assert len(got[s]) == len(want), (s, len(got[s]), len(want))
        for i, (a, b) in enumerate(zip(got[s], want)):
            assert a == b, (s, i, {k: (a[k], b[k]) for k in a if k != "data"}, a["data"] == b["data"])
        total += len(want)
    assert total >= (3 if mode == lib.GRAB_ALL else 1), total


# ---- the reference's decoders ---------------------------------------------------------------------------------------

def decoder_statistics(devices, n=1 << 18):
    """r433b_dispatch_r_devices over every chained call gives the decoded JSON and decode_* counters of the uncut
    mixed batch."""
    if not refh.available():
        pytest.skip("needs the compiled reference (oracle/_ref)")
    kinds = ("silvercrest", "nexus", "nice")
    slots = [[("d0 cu8", synth.ook_stream(60, n_samples=n, n_bursts=3, kinds=kinds, decodable=True), lib.FMT_CU8, 250000,
               433920000)],
             [("d1 cs8", synth.ook_stream(52, n_samples=n, n_bursts=3, kinds=kinds, decodable=True) ^ 0x80, lib.FMT_CS8,
               250000, 433920000),
              ("d1 cs16", synth.fsk_stream(62, n_samples=n // 2, n_bursts=2, rate=1024000), lib.FMT_CS16, 1024000,
               868000000)]]
    r = refh.Ref(chain_decoders=True, store_bitbuffers=False)
    nd = r.register_defaults()
    c = lib.Context(0)
    try:
        c.set_devices(r.registered())
        flat = [f for files in slots for f in files]
        data, offsets, lens = tm._pack(flat)
        c.process_mixed(data, offsets, [f[2] for f in flat], [f[3] for f in flat], [f[4] for f in flat], lengths=lens,
                        block_bytes=BLOCK)
        c.fetch()
        want = [tc._decode(r, c, s, nd) for s in range(len(flat))]
        want = [(want[0][0], want[0][1]), (want[1][0] + want[2][0], want[1][1] + want[2][1])]
        assert sum(len(w[0]) for w in want) >= 3, [len(w[0]) for w in want]
        got = [([], np.zeros_like(want[0][1])) for _ in slots]

        def per_call(cx, res, ch):
            for s in range(len(slots)):
                js, st = tc._decode(r, cx, s, nd)
                got[s] = (got[s][0] + js, got[s][1] + st)

        run_chain(c, slots, [calls_of(slots[0], 1), calls_of(slots[1], 3)], per_call=per_call)
        for s in range(len(slots)):
            assert got[s][0] == want[s][0], f"slot {s}: decoded JSON"
            assert np.array_equal(got[s][1], want[s][1]), f"slot {s}: decode_* counters"
    finally:
        c.close()
        r.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------

def refusals(ctx, devices):
    """Every refusal returns its code and leaves the context and the chain usable and unchanged: the run that follows
    equals one that never saw it."""
    slots = changing_slots(1 << 16)[:2]
    files = [s[0] for s in slots]  # cu8 250k, cs8 250k
    first = [_raw(f[1])[:2 * BLOCK] for f in files]
    rest = [_raw(f[1])[2 * BLOCK:] for f in files]
    fmts, rates, freqs = [f[2] for f in files], [f[3] for f in files], [f[4] for f in files]

    def call(ch, chunks, last, fmts=fmts, rates=rates, freqs=freqs, want_stages=0, chain_h=None, fmt_null=False,
             n_streams=None):
        data, offsets, lens = tm._pack([("", c, f, r, q) for c, f, r, q in zip(chunks, fmts, rates, freqs)])
        lens = np.ascontiguousarray(lens, np.uint64)
        b = lib.Batch(data.ctypes.data, offsets.ctypes.data_as(C.POINTER(C.c_uint64)),
                      len(chunks) if n_streams is None else n_streams, 0, 0, 0, lib.FPDM_AUTO, BLOCK, 0, want_stages,
                      lens.ctypes.data_as(C.POINTER(C.c_uint64)))
        f = (lib.StreamFormat * len(chunks))()
        for i in range(len(chunks)):
            f[i] = lib.StreamFormat(fmts[i], rates[i], freqs[i])
        flags = np.ascontiguousarray(last, np.uint8)
        return ctx.L.r433b_process_mixed_chained(ctx.h, C.byref(b), None if fmt_null else f,
                                                 chain_h if chain_h is not None else ch.h, flags.ctypes.data)

    def finish(ch):
        assert call(ch, rest, [1, 1]) == 0, ctx.L.r433b_last_error(ctx.h)
        res = ctx.fetch()
        pk = res["packages"]
        return [[tuple(int(k[f]) for f in ("seq", "offset", "end_pos", "block")) for k in pk[pk["stream"] == s]]
                for s in range(2)]

    with lib.Chain(ctx, 2) as ch:
        assert call(ch, first, [0, 0]) == 0
        want = finish(ch)
    assert sum(len(w) for w in want) > 0
    other = lib.Context(0)
    try:
        other.set_devices(devices)
        with lib.Chain(other, 2) as foreign:
            cases = [
                ("format change on an open slot", ESTATE,
                 lambda ch: call(ch, first, [0, 0], fmts=[lib.FMT_CU8, lib.FMT_CU8])),
                ("rate change on an open slot", ESTATE,
                 lambda ch: call(ch, first, [0, 0], rates=[250000, 1024000])),
                ("centre frequency across FPDM on an open slot", ESTATE,
                 lambda ch: call(ch, first, [0, 0], freqs=[868000000, freqs[1]])),
                ("r433b_process_chained on open mixed files", ESTATE,
                 lambda ch: ctx.L.r433b_process_chained(ctx.h, C.byref(lib.Batch(
                     first[0].ctypes.data, np.array([0, len(first[0]), 2 * len(first[0])], np.uint64).ctypes.data_as(
                         C.POINTER(C.c_uint64)), 2, lib.FMT_CU8, 250000, 433920000, lib.FPDM_AUTO, BLOCK, 0, 0, None)),
                     ch.h, np.zeros(2, np.uint8).ctypes.data)),
                ("non-final cf32 chunk of one block_bytes, at file starts", EINVAL,
                 lambda ch: call(ch, [first[0][:BLOCK], first[1]], [0, 0], fmts=[lib.FMT_CF32, fmts[1]])),
                ("want_stages", EINVAL, lambda ch: call(ch, rest, [1, 1], want_stages=1)),
                ("n_streams mismatch", EINVAL, lambda ch: call(ch, rest[:1], [1])),
                ("chain of another context", EINVAL, lambda ch: call(ch, rest, [1, 1], chain_h=foreign.h)),
                ("null fmt", EINVAL, lambda ch: call(ch, rest, [1, 1], fmt_null=True)),
            ]
            for tag, code, bad in cases:
                at_start = tag.endswith("at file starts")
                with lib.Chain(ctx, 2) as ch:
                    if not at_start:
                        assert call(ch, first, [0, 0]) == 0
                    assert bad(ch) == code, tag
                    if at_start:
                        assert call(ch, first, [0, 0]) == 0
                    assert finish(ch) == want, f"chain or context changed by: {tag}"
            # a level change while a slot is open
            with lib.Chain(ctx, 2) as ch:
                assert call(ch, first, [0, 0]) == 0
                ctx.set_levels(min_snr=12.0)
                try:
                    assert call(ch, rest, [1, 1]) == ESTATE
                finally:
                    ctx.set_levels()
                assert finish(ch) == want, "chain changed by a refused level change"
            # r433b_process_chained's open files refuse the mixed form; at file starts either form may follow
            with lib.Chain(ctx, 2) as ch:
                d, o, l = tm._pack([("", c, lib.FMT_CU8, 250000, 433920000) for c in first])
                ctx.process(d, o, lib.FMT_CU8, 250000, 433920000, block_bytes=BLOCK, lengths=l, chain=ch, last=[0, 0])
                assert call(ch, first, [0, 0], fmts=[lib.FMT_CU8] * 2, freqs=[433920000] * 2) == ESTATE
                d, o, l = tm._pack([("", c, lib.FMT_CU8, 250000, 433920000) for c in rest])
                ctx.process(d, o, lib.FMT_CU8, 250000, 433920000, block_bytes=BLOCK, lengths=l, chain=ch, last=[1, 1])
                assert call(ch, first, [0, 0]) == 0
                assert finish(ch) == want
    finally:
        other.close()


# ------------------------------------------------------------------------------------------------------- tests ------

@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("blocks", [1, 3, 16])
def test_corpus_parity(ctx, devices, blocks, on_device):
    corpus_parity(ctx, devices, blocks=blocks, on_device=on_device, analyze=blocks == 3)


@pytest.mark.parametrize("fpdm", [lib.FPDM_CLASSIC, lib.FPDM_MINMAX])
def test_forced_fpdm_with_gates(ctx, devices, fpdm):
    corpus_parity(ctx, devices, gates=True, fpdm=fpdm, analyze=False)


def test_descending_offsets(ctx, devices):
    corpus_parity(ctx, devices, blocks=1, reverse=True, analyze=False)


@pytest.mark.parametrize("on_device", [False, True])
def test_order_changes_between_calls(ctx, devices, on_device):
    order_changes(ctx, devices, on_device=on_device)


def test_carried_state(ctx, devices):
    carried_state(ctx, devices)


def test_spoiled_front(devices, monkeypatch):
    spoiled_front(devices, monkeypatch)


def test_arena_overflow(devices, monkeypatch):
    arena_overflow(devices, monkeypatch)


def test_one_format_equals_process_chained(ctx, devices):
    one_format_equals_chained(ctx, devices)


def test_split_chain_runs_unsplit(ctx, devices):
    split_chain_unsplit(ctx, devices)


@pytest.mark.parametrize("on_device", [False, True])
def test_grabbing_chain(ctx, on_device):
    grabbing_chain(ctx, on_device=on_device)


@tg.needs_ref
@pytest.mark.parametrize("mode", ["unknown", "known", "undecoded"])
def test_grab_modes_with_reference_decoders(mode):
    decoders = tg.Decoders()
    c = lib.Context(0)
    try:
        c.set_devices(decoders.devices)
        grabbing_chain(c, mode=tg.MODES[mode], decoders=decoders)
    finally:
        c.close()
        decoders.close()


def test_decoder_statistics(devices):
    decoder_statistics(devices)


def test_refusals(ctx, devices):
    refusals(ctx, devices)
