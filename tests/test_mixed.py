"""-m gpu: mixed batches (include/r433b.h: r433b_process_mixed).  Capture files of different sample formats, rates and
centre frequencies are interleaved in one batch; every stream's results must equal those of its file alone through
r433b_process(), with nothing relaxed: every r433b_package field but the ones that say where it lies (stream mapped),
the pulse and gap widths, every pair's counts and every event, the stream digest, every pulse_data_t field and
sample_file_pos, and the analyzer's text and trial events.  The signal grabber over the interleaved files equals the
stock reference's `rtl_433 -S all -r f1 -r f2 ...` (or tests/golden/grab_mixed.json where it is not built).
tests/test_emu_mixed.py runs the same bodies, smaller, under the SIMT emulator."""
import io
import json
import os
import tempfile

import ctypes as C
import numpy as np
import pytest

import helpers
import test_grab
from rtl_433_b200 import captures, lib, synth
from test_gpu_parity import ctx, devices  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "grab_mixed.json")
BLOCK = 16384  # whole tiles of both sample sizes: several blocks per file at test sizes


def _ook(seed, n, rate):
    for bursts in (2, 1, 0):
        try:
            return synth.ook_stream(seed, n_samples=n, n_bursts=bursts, rate=rate, kinds=("manchester", "silvercrest"))
        except ValueError:
            pass
    raise ValueError("no room")


def corpus(n):
    """[(tag, bytes as uint8, format, rate, centre frequency)], groups interleaved, ragged, with an empty file and one
    shorter than a block."""
    a = _ook(1, n, 250000)
    fsk = synth.fsk_stream(2, n_samples=n, n_bursts=1, rate=1024000)
    return [
        ("cu8_250k", a, lib.FMT_CU8, 250000, 433920000),
        ("cs16_1024k", fsk, lib.FMT_CS16, 1024000, 868000000),
        ("cs8_250k_315M", _ook(3, n - 3000, 250000) ^ 0x80, lib.FMT_CS8, 250000, 315000000),
        ("cu8_2048k", _ook(4, n, 2048000), lib.FMT_CU8, 2048000, 433920000),
        ("cu8_1024k_fsk", synth.fsk_burst_stream(5, 64, n_samples=n, rate=1024000, cu8=True), lib.FMT_CU8, 1024000, 868000000),
        ("empty", np.zeros(0, np.uint8), lib.FMT_CU8, 250000, 433920000),
        ("cf32_1024k", (synth.fsk_stream(6, n_samples=n, n_bursts=1, rate=1024000).astype(np.float32) / 32767.0).astype(np.float32),
         lib.FMT_CF32, 1024000, 868000000),
        ("cu8_250k_b", _ook(7, n - 1000, 250000), lib.FMT_CU8, 250000, 433920000),
        ("cs16_short", fsk[:2 * 3000], lib.FMT_CS16, 1024000, 868000000),
        ("cs16_1024k_b", synth.fsk_stream(8, n_samples=n, n_bursts=1, rate=1024000), lib.FMT_CS16, 1024000, 915000000),
    ]


def _pack(items, reverse=False):
    """-> data, offsets, lengths: every file at a 32-byte aligned start (reverse: placed back to front, so that the
    offsets descend)."""
    raw = [x.view(np.uint8).ravel() for _, x, *_ in items]
    lens = [len(r) for r in raw]
    slots = [(n + 31) // 32 * 32 for n in lens]
    order = list(range(len(raw)))[::-1] if reverse else list(range(len(raw)))
    offsets = np.zeros(len(raw) + 1, np.uint64)
    at = 0
    for i in order:
        offsets[i] = at
        at += slots[i]
    offsets[-1] = at
    data = np.zeros(max(at, 32), np.uint8)
    for i, r in enumerate(raw):
        data[int(offsets[i]):int(offsets[i]) + len(r)] = r
    return data, offsets, lens


def snapshot(ctx, res, s, analyzed):
    """Everything the batch holds for stream s, in a form that does not depend on where the stream sat."""
    pk = res["packages"]
    idx = np.nonzero(pk["stream"] == s)[0]
    fields = [f for f in lib.PACKAGE_DTYPE.names if f not in ("stream", "pulse_off", "first_pair")]
    out = {"headers": [tuple(int(pk[i][f]) for f in fields) for i in idx],
           "pairs": [res["pairs"][int(pk[i]["first_pair"]) // res["n_devices"]].tobytes() if res["n_devices"] else b""
                     for i in idx],
           "results": helpers.gpu_stream_results(ctx, s), "digest": ctx.stream_digest(s)}
    # every pulse_data_t field, and sample_file_pos
    pds = []
    for i in idx:
        pd = ctx.pulse_data(int(i))
        pds.append((bytes(C.string_at(C.addressof(pd), C.sizeof(pd))), ctx.file_pos(int(i))))
    out["pulse_data"] = pds
    if analyzed:
        out["analysis"] = []
        for i in idx:
            a, g, text, bbs = ctx.analysis(int(i))
            out["analysis"].append((bytes(a), bytes(g), text, bbs.tobytes()))
    return out


def _drop_positions(snap):
    """The pair table's event offsets say where in the arena the events lie: compare the rest of every pair."""
    pairs = []
    for p in snap["pairs"]:
        a = np.frombuffer(p, lib.PAIR_DTYPE)
        pairs.append([tuple(int(r[f]) for f in lib.PAIR_DTYPE.names if f != "offset") for r in a])
    snap = dict(snap)
    snap["pairs"] = pairs
    return snap


def alone(ctx, items, fpdm=lib.FPDM_AUTO, analyze=False):
    """Each file by itself through r433b_process() -> one snapshot per file."""
    out = []
    for tag, x, fmt, rate, freq in items:
        data, offsets, lens = _pack([(tag, x, fmt, rate, freq)])
        ctx.process(data, offsets, fmt, rate, freq, fpdm, BLOCK, lengths=lens)
        res = ctx.fetch()
        if analyze:
            ctx.analyze()
        out.append(_drop_positions(snapshot(ctx, res, 0, analyze)))
    return out


def mixed(ctx, items, fpdm=lib.FPDM_AUTO, analyze=False, on_device=False, reverse=False, block_bytes=BLOCK):
    data, offsets, lens = _pack(items, reverse)
    keep = None
    if on_device:
        import torch
        keep = torch.from_numpy(data).cuda()
        data = keep.data_ptr()
    ctx.process_mixed(data, offsets, [t[2] for t in items], [t[3] for t in items], [t[4] for t in items], lengths=lens,
                      fpdm_mode=fpdm, data_on_device=on_device, block_bytes=block_bytes)
    res = ctx.fetch()
    if analyze:
        ctx.analyze()
    snaps = [_drop_positions(snapshot(ctx, res, i, analyze)) for i in range(len(items))]
    del keep
    return snaps, ctx.timing()


def same(got, want, items, tag):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        t = f"{tag} stream {i} ({items[i][0]})"
        d = helpers.compare_results(w["results"], g["results"], t, stages=False)
        assert not d, "\n".join(d[:20])
        for k in w:
            if k != "results":
                assert g[k] == w[k], f"{t}: {k} differs"


def per_stream_parity(ctx, devices, n=1 << 17, on_device=False, gates=False, fpdm=lib.FPDM_AUTO, analyze=True,
                      reverse=False):
    items = corpus(n)
    ctx.set_gates(lib.default_gates(devices) if gates else None)
    try:
        want = alone(ctx, items, fpdm, analyze)
        assert sum(len(w["headers"]) for w in want) > 5, "nothing detected: nothing checked"
        assert any(h[1] == lib.PACKAGE_FSK for w in want for h in w["headers"]), "no FSK package"
        got, tm = mixed(ctx, items, fpdm, analyze, on_device, reverse)
    finally:
        ctx.set_gates(None)
    same(got, want, items, f"mixed fpdm={fpdm} gates={gates} device={on_device}")
    # classes: (250k cu8), (250k cs8), (1024k cu8), (1024k cs16, 868M and 915M, cf32 converted), (2048k cu8)
    assert tm["mixed_classes"] == 5, tm
    assert tm["detect_launches"] == tm["mixed_classes"] + (1 if on_device else 0), tm
    return tm


def homogeneous(ctx, devices, n=1 << 17):
    """One format through r433b_process_mixed equals r433b_process, digests and grabs included."""
    items = [t for t in corpus(n) if t[2] == lib.FMT_CU8 and t[3] == 250000]
    data, offsets, lens = _pack(items)
    ctx.process(data, offsets, lib.FMT_CU8, 250000, 433920000, lib.FPDM_AUTO, BLOCK, lengths=lens)
    ctx.fetch()
    want = [ctx.stream_digest(i) for i in range(len(items))]
    plan = ctx.grab_plan(lib.GRAB_ALL)
    want_grab = (plan.tobytes(), ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes(), ctx.grab_tail()[1].tobytes())
    ctx.process_mixed(data, offsets, [lib.FMT_CU8] * len(items), [250000] * len(items), [433920000] * len(items),
                      lengths=lens, block_bytes=BLOCK)
    ctx.fetch()
    assert [ctx.stream_digest(i) for i in range(len(items))] == want
    plan = ctx.grab_plan(lib.GRAB_ALL)
    got_grab = (plan.tobytes(), ctx.grab_copy(0, len(plan), int(plan["bytes"].sum())).tobytes(), ctx.grab_tail()[1].tobytes())
    assert got_grab == want_grab
    assert ctx.timing()["mixed_classes"] == 1


def arena_overflow(devices, monkeypatch, n=1 << 16):
    """Package and pool arenas far too small: every class runs again with the caps the device counted."""
    items = corpus(n)
    c = lib.Context(0)
    c.set_devices(devices)
    want = alone(c, items)
    c.close()
    monkeypatch.setenv("R433B_TEST_CAPS", "4,64,256")
    c = lib.Context(0)
    try:
        c.set_devices(devices)
        got, tm = mixed(c, items)
        same(got, want, items, "overflow")
    finally:
        c.close()


def refusals(ctx, devices, n=1 << 16):
    items = corpus(n)[:4]
    data, offsets, lens = _pack(items)
    fmts, rates, freqs = [t[2] for t in items], [t[3] for t in items], [t[4] for t in items]

    def call(**kw):
        b = lib.Batch(data.ctypes.data, np.ascontiguousarray(kw.get("offsets", offsets), np.uint64).ctypes.data_as(C.POINTER(C.c_uint64)),
                      len(items), kw.get("sample_format", 0), kw.get("samp_rate", 0), 0, lib.FPDM_AUTO, kw.get("block_bytes", BLOCK),
                      0, kw.get("want_stages", 0), None)
        f = (lib.StreamFormat * len(items))()
        for i in range(len(items)):
            f[i] = lib.StreamFormat(kw.get("fmts", fmts)[i], kw.get("rates", rates)[i], freqs[i])
        return ctx.L.r433b_process_mixed(ctx.h, C.byref(b), f)

    assert call() == 0
    for kw in ({"sample_format": lib.FMT_CU8}, {"samp_rate": 250000}, {"want_stages": 1},
               {"rates": [250000, 0, 250000, 2048000]}, {"fmts": [lib.FMT_CU8, 7, lib.FMT_CS8, lib.FMT_CU8]},
               {"block_bytes": 4096},  # 2048 samples of cu8 but not of the cs16 stream
               {"offsets": offsets + np.array([0, 8, 0, 0, 0], np.uint64)},
               {"fmts": [lib.FMT_CU8, lib.FMT_CF32, lib.FMT_CS8, lib.FMT_CU8],
                "offsets": offsets + np.array([0, 16, 16, 16, 16], np.uint64)}):
        assert call(**kw) == -1, kw
        assert call() == 0, f"context unusable after {kw}"
    # no chained form: the Python binding has none, and the C call takes no chain
    ctx.process_mixed(data, offsets, fmts, rates, freqs, lengths=lens, block_bytes=BLOCK)
    ctx.fetch()


# ---- the signal grabber and the command line, at the reference's block size ------------------------------------------

def grab_case():
    """[(file name, bytes)] in command-line order: groups interleaved, sample sizes alternating so that windows reach
    back into an earlier file of another sample size, a file shorter than one block and one without signal."""
    def ook(seed, n, bursts):
        return synth.ook_stream(seed, n_samples=n, n_bursts=bursts, kinds=("silvercrest", "nexus"))
    fsk = [synth.fsk_stream(310 + i, n_samples=1 << 18, n_bursts=2, rate=1024000) for i in range(2)]
    return [("m0_433.92M_250k.cu8", ook(301, 60000, 1).tobytes()),
            ("m1_868M_1024k.cs16", fsk[0].tobytes()),
            ("m2_315M_250k.cs8", test_grab._cs8(ook(302, 1 << 18, 2)).tobytes()),
            ("m3_868M_1024k.cf32", test_grab._cf32(fsk[1]).tobytes()),
            ("m4_433.92M_250k.cu8", ook(303, 40000, 0).tobytes()),
            ("m5_433.92M_2048k.cu8", ook(304, 1 << 19, 2).tobytes()),
            ("m6_915M_1024k.cs16", synth.fsk_stream(312, n_samples=1 << 18, n_bursts=2, rate=1024000).tobytes())]


def gpu_grabs_mixed(ctx, paths, on_device=False):
    err = io.StringIO()
    batch = captures.load_batches(paths, one_batch=True)[0]
    ss = {"cu8": 2, "cs8": 2, "cs16": 4, "cf32": 4}
    with tempfile.TemporaryDirectory() as d:
        g = captures.Grabber(d, err=err)
        keep, data = None, batch["data"]
        if on_device:
            import torch
            keep = torch.from_numpy(data).cuda()
            data = keep.data_ptr()
        ctx.process_mixed(data, batch["offsets"], batch["abi_formats"], batch["rates"], batch["freqs"],
                          lengths=batch["lengths"], data_on_device=on_device)
        ctx.fetch()
        g.write(ctx, lib.GRAB_ALL, None, None, None,
                per_stream=[(f, r, ss[t]) for f, r, t in zip(batch["freqs"], batch["rates"], batch["formats"])])
        del keep
        files = {}
        for name in sorted(os.listdir(d)):
            with open(os.path.join(d, name), "rb") as f:
                files[name] = f.read()
    return files


def grab_vs_reference(ctx, devices, on_device=False):
    ctx.set_devices(devices)
    with tempfile.TemporaryDirectory() as d:
        paths = test_grab.write_case(grab_case(), d)
        got = gpu_grabs_mixed(ctx, paths, on_device)
        assert len(got) >= 4, sorted(got)
        assert {n.rsplit(".", 1)[1] for n in got} == {"cu8", "cs16"}, sorted(got)
        if os.path.exists(test_grab.CLI):
            want, _ = test_grab.reference_grabs(paths, "all")
            assert sorted(got) == sorted(want)
            for name in want:
                assert got[name] == want[name], f"{name} differs from the reference's"
        else:
            with open(GOLDEN) as f:
                assert test_grab.fingerprint(got) == json.load(f)["all"]


def command_line(ctx, devices, capsys):
    with tempfile.TemporaryDirectory() as d:
        paths = test_grab.write_case(grab_case(), d)
        plain = captures.replay(paths, out=lambda *a: None)
        one = captures.replay(paths, out=lambda *a: None, one_batch=True)
        assert sorted(plain, key=lambda r: r["file"]) == sorted(one, key=lambda r: r["file"])
        assert [r["file"] for r in one] == paths
        gdir = os.path.join(d, "grabs")
        os.mkdir(gdir)
        captures.replay(paths, out=lambda *a: None, one_batch=True, grab_mode=lib.GRAB_ALL, grab_dir=gdir)
        got = {}
        for name in sorted(os.listdir(gdir)):
            with open(os.path.join(gdir, name), "rb") as f:
                got[name] = f.read()
        assert got == gpu_grabs_mixed(ctx, paths)
    for bad in (["--one-batch", "--chunk-mb", "4", "x.cu8"], ["--one-batch", "--split", "x.cu8"]):
        with pytest.raises(SystemExit):
            captures.main(bad)
    with pytest.raises(ValueError):
        captures.replay(["x.cu8"], one_batch=True, chunk_mb=4)


# ------------------------------------------------------------------------------------------------------- tests ------

@pytest.mark.parametrize("on_device", [False, True])
def test_per_stream_parity(ctx, devices, on_device):
    per_stream_parity(ctx, devices, on_device=on_device)


@pytest.mark.parametrize("fpdm", [lib.FPDM_CLASSIC, lib.FPDM_MINMAX])
def test_forced_fpdm_with_gates(ctx, devices, fpdm):
    per_stream_parity(ctx, devices, gates=True, fpdm=fpdm, analyze=False)


def test_descending_offsets(ctx, devices):
    per_stream_parity(ctx, devices, reverse=True, analyze=False)


def test_homogeneous_equals_process(ctx, devices):
    homogeneous(ctx, devices)


def test_arena_overflow(devices, monkeypatch):
    arena_overflow(devices, monkeypatch)


def test_refusals(ctx, devices):
    refusals(ctx, devices)


@pytest.mark.parametrize("on_device", [False, True])
def test_grab_vs_reference(ctx, devices, on_device):
    grab_vs_reference(ctx, devices, on_device)


def test_command_line(ctx, devices, capsys):
    command_line(ctx, devices, capsys)
