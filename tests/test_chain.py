"""-m gpu: chained batches (include/r433b.h: r433b_process_chained).  A file cut into chunks at whole-block boundaries
and passed chunk by chunk through a chain must give exactly what the uncut file gives: package headers (absolute
offset and block, start_ago / end_ago, sample_file_pos), pulse and gap widths, every event, and the stage arrays.
tests/test_emu_chain.py runs the same bodies under the SIMT emulator.

Which case covers which piece of the device side (r433b_front.cuh, r433b_detect.cuh):
  * tile 0 of a continued chunk starts from the carried AM state (k_front) and is checked against it (k_detect's
    hand-over at t0 == 0): every case; spoiled_first_tiles makes the guess wrong so the check must repair it;
  * the IQ sample in front of the chunk (disc_fill) and the carried FM state (fm_cold, the stage pass):
    fsk_cs16_cut_in_first_pulses (monotone and wrapping filters, with stage arrays), cs8_and_cf32;
  * the chunk end (log fold, exact FM state, last IQ sample): long_ook_package_folded_at_boundaries, fsk_cs16_...;
  * positions across a boundary (start_abs, fsk_offset, FmState.pos, package offset): every case with a package that
    spans a boundary; per-stream start and both launch paths: ragged_slots, time_sliced_chains."""
import numpy as np
import pytest

import helpers
from oracle import refh
from rtl_433_b200 import lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OOK_RATE, FSK_RATE = 250000, 1024000
WRAPPING = 0.6  # -Y ratio above 0.5: a filter that is not provably monotone


def _in_bytes(fmt):
    return 8 if fmt == lib.FMT_CF32 else fmt & 0xff


def _pack(chunks):
    """Chunks (uint8 arrays) -> (data, offsets, lengths) with every stream start 32-byte aligned."""
    lens = [len(c) for c in chunks]
    stride = [(n + 31) // 32 * 32 for n in lens]
    offsets = np.concatenate([[0], np.cumsum(stride)]).astype(np.uint64)
    data = np.zeros(max(int(offsets[-1]), 32), np.uint8)
    for c, o in zip(chunks, offsets[:-1]):
        data[int(o):int(o) + len(c)] = c
    return data, offsets, lens


def _empty():
    return {"packages": [], "events": [], "am": [], "fm": [], "hdr": []}


def _add(acc, ctx, res, i, n_samples, stages):
    # seq and end_pos are not among compare_results' keys: compared here directly
    pk = res["packages"][res["packages"]["stream"] == i]
    acc["hdr"] += [(int(k["seq"]), int(k["end_pos"])) for k in pk]
    got = helpers.gpu_stream_results(ctx, i)
    k0 = len(acc["packages"])
    acc["packages"] += got["packages"]
    for e in got["events"]:
        e["package"] += k0
        acc["events"].append(e)
    if stages:
        am, fm = ctx.copy_stage(i, n_samples) if n_samples else (np.zeros(0, np.int16),) * 2
        acc["am"].append(am)
        acc["fm"].append(fm)


def _finish(acc, stages):
    if stages:
        acc["am"] = np.concatenate(acc["am"]) if acc["am"] else np.zeros(0, np.int16)
        acc["fm"] = np.concatenate(acc["fm"]) if acc["fm"] else np.zeros(0, np.int16)
    else:
        del acc["am"], acc["fm"]
    return acc


def run_uncut(ctx, files, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, stages=False):
    """Every file whole, one stream each, in one batch."""
    data, offsets, lens = _pack([f.view(np.uint8).ravel() for f in files])
    ctx.process(data, offsets, fmt, rate, freq, fpdm, block_bytes, want_stages=stages, lengths=lens)
    res = ctx.fetch()
    out = []
    for i, n in enumerate(lens):
        acc = _empty()
        _add(acc, ctx, res, i, n // _in_bytes(fmt), stages)
        out.append(_finish(acc, stages))
    run_uncut.timing = ctx.timing()
    return out


def run_chained(ctx, slots, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, stages=False):
    """slots[i] = the files of slot i in order, each a list of chunks (uint8 arrays).  Round r passes every slot's next
    chunk; a slot without one gets an empty last chunk (a new empty file, not collected).
    -> ([[result per file] per slot], summed counters)"""
    queues = [[(c, j == len(f) - 1, fi) for fi, f in enumerate(files) for j, c in enumerate(f)] for files in slots]
    out = [[_empty() for _ in files] for files in slots]
    totals = {k: 0 for k in ("chain_folds", "chain_fm_rebuilds", "front_repairs", "idle_skipped", "detect_launches")}
    chain = lib.Chain(ctx, len(slots))
    try:
        for r in range(max(len(q) for q in queues)):
            items = [q[r] if r < len(q) else (np.zeros(0, np.uint8), True, None) for q in queues]
            data, offsets, lens = _pack([c for c, _, _ in items])
            ctx.process(data, offsets, fmt, rate, freq, fpdm, block_bytes, want_stages=stages, lengths=lens, chain=chain,
                        last=[int(last) for _, last, _ in items])
            res = ctx.fetch()
            tm = ctx.timing()
            for k in totals:
                totals[k] += tm[k]
            for i, (c, _, fi) in enumerate(items):
                if fi is not None:
                    _add(out[i][fi], ctx, res, i, len(c) // _in_bytes(fmt), stages)
    finally:
        chain.close()
    return [[_finish(a, stages) for a in files] for files in out], totals


def cut(x, block, at):
    """Chunks of the bytes of x at the whole-block boundaries `at` (block indices)."""
    b = x.view(np.uint8).ravel()
    edges = [0] + [k * block for k in at if 0 < k * block < len(b)] + [len(b)]
    return [b[edges[j]:edges[j + 1]] for j in range(len(edges) - 1)]


def every_block(x, block):
    return cut(x, block, range(1, len(x.view(np.uint8).ravel()) // block + 1))


def check(got, want, tag, stages=True):
    d = helpers.compare_results(want, got, tag, stages=stages)
    assert not d, "\n".join(d[:20])
    if "hdr" in got and "hdr" in want:
        assert got["hdr"] == want["hdr"], f"{tag}: (seq, end_pos) {got['hdr'][:8]} != {want['hdr'][:8]}"


def vs_reference(want, files, ss, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, low_pass=0.0, tag=""):
    """The uncut runs against the compiled reference, where it is present (guards against both runs being wrong)."""
    if not refh.available():
        return
    r = refh.Ref(store_bitbuffers=False, store_stages=False)
    r.register_defaults()
    if low_pass:
        r.set_fm_low_pass(low_pass)
    for i, f in enumerate(files):
        check({k: v for k, v in want[i].items() if k != "hdr"}, r.run(f, ss, rate, freq, fpdm, block_bytes),
              f"{tag} uncut file {i} vs reference", stages=False)


def compare(ctx, files, chunked, fmt, rate, freq=433920000, fpdm=lib.FPDM_AUTO, block_bytes=0, stages=True, tag="",
            spoiled=False):
    """Chained (one slot per file) against uncut; returns the chained run's counters.  Unspoiled, tile 0 of a continued
    chunk starts from the exact carried state and never needs a repair: the chained run repairs at most the tiles the
    uncut run repairs (a wrong carried state would be repaired silently, so only this count shows it)."""
    want = run_uncut(ctx, files, fmt, rate, freq, fpdm, block_bytes, stages)
    uncut_repairs = run_uncut.timing["front_repairs"]
    got, tm = run_chained(ctx, [[c] for c in chunked], fmt, rate, freq, fpdm, block_bytes, stages)
    for i in range(len(files)):
        assert want[i]["packages"], f"{tag} file {i}: no packages, nothing checked"
        check(got[i][0], want[i], f"{tag} file {i}", stages)
    if not spoiled:
        assert tm["front_repairs"] <= uncut_repairs, (tag, tm, uncut_repairs)
    return tm, want


# ------------------------------------------------------------------------------------------------------- cases ------

def ook_cu8_every_and_random_boundaries(ctx, devices):
    """Every 4 KiB block boundary (boundaries in packages, in GAPs waiting for their end, in idle runs), then random
    whole-block boundaries of 4 KiB blocks with skipped idle runs on both sides of them; the uncut run against the
    compiled reference where it is present."""
    files = [synth.ook_stream(k, n_samples=1 << 16, n_bursts=3) for k in (700, 705)]
    compare(ctx, files, [every_block(f, 4096) for f in files], lib.FMT_CU8, OOK_RATE, block_bytes=4096, tag="every block")
    rng = np.random.default_rng(7)
    long_files = [synth.ook_stream(k, n_samples=1 << 18, n_bursts=2) for k in (710, 714)]
    chunked = [cut(f, 4096, sorted(rng.choice(np.arange(1, 128), 9, replace=False))) for f in long_files]
    tm, want = compare(ctx, long_files, chunked, lib.FMT_CU8, OOK_RATE, block_bytes=4096, stages=False, tag="random")
    assert tm["idle_skipped"] > 0, tm
    vs_reference(want, long_files, 2, OOK_RATE, block_bytes=4096, tag="random")


def test_ook_cu8_every_and_random_boundaries(ctx, devices):
    ook_cu8_every_and_random_boundaries(ctx, devices)


def fsk_cs16_cut_in_first_pulses(ctx, devices):
    """cs16 2-FSK cut at every 16 KiB block: boundaries inside the first pulse of every package while the FSK
    sub-detector runs; minmax and classic, a monotone and a wrapping FM filter, with stage arrays."""
    files = [synth.fsk_stream(720 + k, n_samples=1 << 17, n_bursts=2) for k in range(2)]
    for low_pass in (0.0, WRAPPING):
        ctx.set_fm_low_pass(low_pass)
        try:
            for fpdm, freq in ((lib.FPDM_AUTO, 868000000), (lib.FPDM_CLASSIC, 433920000)):
                tm, want = compare(ctx, files, [every_block(f, 16384) for f in files], lib.FMT_CS16, FSK_RATE, freq, fpdm,
                                   block_bytes=16384, tag=f"fsk fpdm {fpdm} low-pass {low_pass}")
                assert any(p["type"] == 2 for w in want for p in w["packages"])
                assert tm["chain_fm_rebuilds"] > 0, tm
                vs_reference(want, files, 4, FSK_RATE, freq, fpdm, 16384, low_pass, tag=f"fsk fpdm {fpdm}")
        finally:
            ctx.set_fm_low_pass(0.0)


def test_fsk_cs16_cut_in_first_pulses(ctx, devices):
    fsk_cs16_cut_in_first_pulses(ctx, devices)


def long_ook_package_folded_at_boundaries(ctx, devices):
    """A long OOK package (FM on: the default devices include FSK ones) cut at every block: its deferred carrier
    estimate is folded at every boundary inside it."""
    files = [synth.ook_train_stream(730, n_pulses=300, n_samples=1 << 16)]
    tm, want = compare(ctx, files, [every_block(f, 4096) for f in files], lib.FMT_CU8, OOK_RATE, block_bytes=4096,
                       tag="long package")
    assert tm["chain_folds"] > 0, tm
    vs_reference(want, files, 2, OOK_RATE, block_bytes=4096, tag="long package")


def test_long_ook_package_folded_at_boundaries(ctx, devices):
    long_ook_package_folded_at_boundaries(ctx, devices)


def spoiled_first_tiles(devices, monkeypatch):
    """R433B_SPOIL_FRONT=4 also spoils tile 0 of every continued chunk: k_detect's hand-over check at t0 == 0 must find
    and repair it."""
    monkeypatch.setenv("R433B_SPOIL_FRONT", "4")
    c = lib.Context(0)
    monkeypatch.delenv("R433B_SPOIL_FRONT")
    try:
        c.set_devices(devices)
        files = [synth.ook_stream(743, n_samples=1 << 16, n_bursts=3)]
        chunked = [every_block(f, 4096) for f in files]
        tm, _ = compare(c, files, chunked, lib.FMT_CU8, OOK_RATE, block_bytes=4096, tag="spoiled", spoiled=True)
        assert tm["front_repairs"] >= len(chunked[0]) - 1, tm
    finally:
        c.close()


def test_spoiled_first_tiles(devices, monkeypatch):
    spoiled_first_tiles(devices, monkeypatch)


def cs8_and_cf32(ctx, devices):
    """cs8 (cu8 - 128) and cf32 (cs16 / 32767) input cut at every block."""
    ook = synth.ook_stream(702, n_samples=1 << 16, n_bursts=1)
    cs8 = (ook.astype(np.int16) - 128).astype(np.int8)
    _, want = compare(ctx, [cs8], [every_block(cs8, 4096)], lib.FMT_CS8, OOK_RATE, block_bytes=4096, tag="cs8")
    vs_reference(want, [ook], 2, OOK_RATE, block_bytes=4096, tag="cs8 (as the cu8 it is read as)")
    fsk = synth.fsk_stream(751, n_samples=1 << 16, n_bursts=1)
    cf32 = (fsk.astype(np.float32) / np.float32(32767.0)).astype(np.float32)
    compare(ctx, [cf32], [every_block(cf32, 2 * 8192)], lib.FMT_CF32, FSK_RATE, 868000000, block_bytes=8192, tag="cf32")


def test_cs8_and_cf32(ctx, devices):
    cs8_and_cf32(ctx, devices)


def ragged_slots(ctx, devices):
    """Slots whose files end in different rounds, empty chunks that are not the last, an empty last chunk (flush
    only), and a slot that starts a second file after its first one's last chunk."""
    blk = 4096
    a = synth.ook_stream(704, n_samples=1 << 16, n_bursts=2)  # 32 blocks
    b = synth.ook_stream(701, n_samples=1 << 15, n_bursts=1)
    c = synth.ook_stream(702, n_samples=1 << 15, n_bursts=1)
    d = synth.ook_stream(703, n_samples=(1 << 15) + 8 * 37, n_bursts=1)  # ragged end
    empty = np.zeros(0, np.uint8)
    ca = cut(a, blk, [3, 4, 9, 20])
    ca = ca[:2] + [empty] + ca[2:]                      # an empty chunk in the middle
    cb = cut(b, blk, [2, 5]) + [empty]                  # an empty last chunk: flush only
    slots = [[ca], [cb], [cut(c, blk, [1, 6]), cut(d, blk, [5])]]  # slot 2: a second file after the first
    got, _ = run_chained(ctx, slots, lib.FMT_CU8, OOK_RATE, block_bytes=blk, stages=True)
    want = run_uncut(ctx, [a, b, c, d], lib.FMT_CU8, OOK_RATE, block_bytes=blk, stages=True)
    for (s, fi), w in zip(((0, 0), (1, 0), (2, 0), (2, 1)), want):
        assert w["packages"]
        check(got[s][fi], w, f"slot {s} file {fi}")
    vs_reference(want, [a, b, c, d], 2, OOK_RATE, block_bytes=blk, tag="ragged")


def test_ragged_slots(ctx, devices):
    ragged_slots(ctx, devices)


def time_sliced_chains(ctx, devices):
    """Chained batches through the time-sliced path (uniform stride) equal the sequential path."""
    files = [synth.ook_stream(k, n_samples=1 << 17, n_bursts=3) for k in (703, 704, 708)]
    chunked = [cut(f, 4096, [16, 32, 48]) for f in files]  # every round: 16 blocks per slot
    try:
        ctx.set_pipeline(1)
        seq, _ = run_chained(ctx, [[c] for c in chunked], lib.FMT_CU8, OOK_RATE, block_bytes=4096)
        ctx.set_pipeline(4)
        sliced, tm = run_chained(ctx, [[c] for c in chunked], lib.FMT_CU8, OOK_RATE, block_bytes=4096)
    finally:
        ctx.set_pipeline(0)
    assert tm["detect_launches"] > 4 * 2, tm
    want = run_uncut(ctx, files, lib.FMT_CU8, OOK_RATE, block_bytes=4096)
    for i in range(len(files)):
        assert want[i]["packages"]
        check(seq[i][0], want[i], f"sequential file {i}", stages=False)
        check(sliced[i][0], want[i], f"time-sliced file {i}", stages=False)


def test_time_sliced_chains(ctx, devices):
    time_sliced_chains(ctx, devices)


def errors(ctx, devices):
    """Lengths that are not whole blocks, a settings change on an open chain, a wrong n_streams, the grabber."""
    x = synth.ook_stream(702, n_samples=1 << 15, n_bursts=1).ravel()
    chain = lib.Chain(ctx, 1)
    try:
        with pytest.raises(lib.R433Error, match="error -1"):
            ctx.process(x[:4096 + 32], [0, 4096 + 32], lib.FMT_CU8, OOK_RATE, block_bytes=4096, chain=chain, last=[0])
        ctx.process(x[:4096], [0, 4096], lib.FMT_CU8, OOK_RATE, block_bytes=4096, chain=chain, last=[0])
        ctx.fetch()
        with pytest.raises(lib.R433Error, match="error -5"):
            ctx.grab_plan(lib.GRAB_ALL)
        with pytest.raises(lib.R433Error, match="error -1"):
            ctx.process(np.concatenate([x[:4096]] * 2), [0, 4096, 8192], lib.FMT_CU8, OOK_RATE, block_bytes=4096,
                        chain=chain, last=[0, 0])
        for change in ({"samp_rate": 2 * OOK_RATE}, {"block_bytes": 8192}, {"center_frequency": 868000000}):
            kw = dict(samp_rate=OOK_RATE, block_bytes=4096, center_frequency=433920000) | change
            with pytest.raises(lib.R433Error, match="error -5"):
                ctx.process(x[4096:8192], [0, 4096], lib.FMT_CU8, chain=chain, last=[0], **kw)
        ctx.set_levels(min_level=-10.0)
        try:
            with pytest.raises(lib.R433Error, match="error -5"):
                ctx.process(x[4096:8192], [0, 4096], lib.FMT_CU8, OOK_RATE, block_bytes=4096, chain=chain, last=[0])
        finally:
            ctx.set_levels()
        # the chain is still usable: the file goes on and ends
        ctx.process(x[4096:], [0, len(x) - 4096], lib.FMT_CU8, OOK_RATE, block_bytes=4096, chain=chain, last=[1])
        assert chain.base(0) == 2048
        # closed: any settings are accepted again, and the slot starts at 0
        ctx.process(x, [0, len(x)], lib.FMT_CU8, 2 * OOK_RATE, block_bytes=8192, chain=chain, last=[1])
        assert chain.base(0) == 0
    finally:
        chain.close()


def test_errors(ctx, devices):
    errors(ctx, devices)


def _decode(r, ctx, s, n):
    """Stream s of the fetched batch through the reference's decoders (r433b_dispatch_r_devices) -> (JSON lines, stats)."""
    import ctypes as C
    ptrs = r.L.refh_begin_external_dispatch(r.h)
    try:
        rc = ctx.L.r433b_dispatch_r_devices(ctx.h, C.byref(ctx._res), s, ptrs, n)
        assert rc == 0, ctx.L.r433b_last_error(ctx.h)
        return ([l for l in r.L.refh_json(r.h).decode().split("\n") if l],
                np.array([r.device_stats(i) for i in range(n)], np.int64))
    finally:
        r.L.refh_end_external_dispatch(r.h)


def _texts(ctx, res, s):
    ctx.analyze()
    return [ctx.analysis(int(i))[2] for i in np.nonzero(res["packages"]["stream"] == s)[0]]


def decoders_and_analyzer(devices):
    """The reference's decoders behind r433b_dispatch_r_devices, ungated and gated: decoded JSON, the decode_* counters,
    sample_file_pos and the analyzer's text of a chained run equal those of the uncut run (and of the reference)."""
    if not refh.available():
        pytest.skip("needs the compiled reference (oracle/_ref)")
    kinds = ("silvercrest", "nexus", "nice")
    files = [synth.ook_stream(50 + i, n_samples=1 << 18, n_bursts=3, kinds=kinds, decodable=True) for i in range(3)]
    blk = 16384
    chunked = [cut(f, blk, at) for f, at in zip(files, ([5, 11, 20, 27], [1, 2, 3, 16], [30]))]
    r = refh.Ref(chain_decoders=True, store_bitbuffers=False)
    n = r.register_defaults()
    devs = r.registered()
    ref_json = [r.run(f, 2, OOK_RATE, 433920000, lib.FPDM_AUTO, blk)["json"] for f in files]
    r.L.refh_reset_stats(r.h)
    with _ctx(devs) as c:
        for gated in (False, True):
            c.set_gates(lib.default_gates(devs) if gated else None)
            data, offsets, lens = _pack([f.view(np.uint8).ravel() for f in files])
            c.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=blk, lengths=lens)
            res = c.fetch()
            want = []
            for s in range(len(files)):
                js, st = _decode(r, c, s, n)
                want.append((js, st, [c.file_pos(int(i)) for i in np.nonzero(res["packages"]["stream"] == s)[0]],
                             _texts(c, res, s)))
            assert [w[0] for w in want] == ref_json and sum(len(w[0]) for w in want) >= 3
            got = [([], np.zeros((n, 8), np.int64), [], []) for _ in files]
            with lib.Chain(c, len(files)) as chain:
                for rd in range(max(len(x) for x in chunked)):
                    items = [x[rd] if rd < len(x) else np.zeros(0, np.uint8) for x in chunked]
                    data, offsets, lens = _pack(items)
                    last = [int(rd >= len(x) - 1) for x in chunked]
                    c.process(data, offsets, lib.FMT_CU8, OOK_RATE, block_bytes=blk, lengths=lens, chain=chain, last=last)
                    res = c.fetch()
                    for s in range(len(files)):
                        if rd >= len(chunked[s]):
                            continue
                        js, st = _decode(r, c, s, n)
                        g = got[s]
                        g[0].extend(js)
                        g[2].extend(c.file_pos(int(i)) for i in np.nonzero(res["packages"]["stream"] == s)[0])
                        g[3].extend(_texts(c, res, s))
                        got[s] = (g[0], g[1] + st, g[2], g[3])
            for s in range(len(files)):
                tag = f"{'gated' if gated else 'ungated'} file {s}"
                assert got[s][0] == want[s][0], tag + ": decoded JSON"
                assert np.array_equal(got[s][1], want[s][1]), tag + ": decode_* counters"
                assert got[s][2] == want[s][2], tag + ": package_file_pos"
                assert got[s][3] == want[s][3], tag + ": analyzer text"


class _ctx:
    def __init__(self, devs):
        self.c = lib.Context(0)
        self.c.set_devices(devs)

    def __enter__(self):
        return self.c

    def __exit__(self, *exc):
        self.c.close()


def test_decoders_and_analyzer(devices):
    decoders_and_analyzer(devices)


def command_line_chunks(capsys, tmp_path):
    """`python -m rtl_433_b200.captures FILES --chunk-mb 1` prints what the plain run prints, for files longer than one
    chunk and of different lengths (cu8 and cs16 groups); -S with --chunk-mb is refused."""
    from rtl_433_b200 import captures
    files = {"a_433.92M_250k.cu8": synth.ook_stream(704, n_samples=(1 << 19) + 77777, n_bursts=3),
             "b_433.92M_250k.cu8": synth.ook_stream(708, n_samples=1 << 20, n_bursts=3),
             "c_433.92M_250k.cu8": synth.ook_stream(702, n_samples=1 << 16, n_bursts=1),
             "f_868M_1024k.cs16": synth.fsk_stream(720, n_samples=(1 << 18) + 1000, n_bursts=3)}
    paths = []
    for name, arr in files.items():
        arr.tofile(tmp_path / name)
        paths.append(str(tmp_path / name))
    captures.main(paths)
    plain = capsys.readouterr().out
    captures.main(paths + ["--chunk-mb", "1"])
    chunked = capsys.readouterr().out
    assert plain.count("package(s)") == 4 and "OOK package" in plain and "FSK package" in plain
    assert chunked == plain
    with pytest.raises(SystemExit):
        captures.main(paths + ["--chunk-mb", "1", "-S", "all"])
    assert "-S does not run with --chunk-mb" in capsys.readouterr().err


def test_command_line_chunks(capsys, tmp_path):
    command_line_chunks(capsys, tmp_path)
