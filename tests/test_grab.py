"""Signal grabber (`rtl_433 -S all|unknown|known|undecoded`, src/samp_grab.c, src/r_flow.c:345-362).

Every file name and every byte the GPU path writes equals what the stock reference program (oracle/_ref/rtl_433)
writes for the same capture files, and the committed fingerprints of those files (tests/golden/grab.json, written
by tools/make_golden_grab.py) where the reference is not built.  The bodies take the library as it is loaded, so
tests/test_emu_grab.py runs them with k_grab under the SIMT emulator."""
import ctypes as C
import hashlib
import io
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import refh
from rtl_433_b200 import captures, lib, synth

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "rtl_433")
GOLDEN = os.path.join(HERE, "golden", "grab.json")
MODES = {"all": lib.GRAB_ALL, "unknown": lib.GRAB_UNKNOWN, "known": lib.GRAB_KNOWN, "undecoded": lib.GRAB_UNDECODED}
KINDS = ("silvercrest", "nexus", "nice")


def _cs8(x):
    return (x ^ 0x80).astype(np.uint8)


def _cf32(x16):
    return (x16.astype(np.float32) / 32767.0).astype(np.float32)


def cases():
    """name -> [(file name, bytes)] in command-line order.  Sizes are chosen so that: the first file is shorter than
    one grab block (its frame is closed by the flush and its window clamped to what was pushed, reaching into
    never-written ring bytes); later frames reach back into the previous file; the run passes the 3 MiB ring, so
    windows wrap in it."""
    def ook(seed, n, bursts, decodable, kinds=KINDS):
        return synth.ook_stream(seed, n_samples=n, n_bursts=bursts, kinds=kinds if decodable else None, decodable=decodable)
    run = [ook(201, 60000, 1, True, ("nice",))] + [ook(202 + i, 1 << 18, 2, i % 2 == 0) for i in range(7)]
    run.insert(3, ook(250, 40000, 0, False))  # no signal; moves the later windows onto the ring's wrap
    out = {"ook_cu8": [("f%d_433.92M_250k.cu8" % i, x.tobytes()) for i, x in enumerate(run)],
           "ook_cs8": [("f%d_433.92M_250k.cs8" % i, _cs8(x).tobytes()) for i, x in enumerate(run[:3])]}
    fsk = [synth.fsk_stream(211 + i, n_samples=1 << 18, n_bursts=2) for i in range(3)]
    out["fsk_cs16"] = [("f%d_868M_1024k.cs16" % i, x.tobytes()) for i, x in enumerate(fsk)]
    out["fsk_cf32"] = [("f%d_868M_1024k.cf32" % i, _cf32(x).tobytes()) for i, x in enumerate(fsk)]
    return out


def fingerprint(files):
    """[name, size, sha256 prefix] of every file, sorted by name."""
    return [[n, len(b), hashlib.sha256(b).hexdigest()[:32]] for n, b in sorted(files.items())]


def write_case(files, directory):
    paths = []
    for name, data in files:
        p = os.path.join(directory, name)
        with open(p, "wb") as f:
            f.write(data)
        paths.append(p)
    return paths


def reference_grabs(paths, mode):
    """The stock rtl_433 with -S `mode` on the files -> {name: bytes}, stderr "Saving" lines.  Its ring is a fresh
    3 MiB malloc(), which the C library maps as new zero pages: bytes the run never wrote read zero there too."""
    with tempfile.TemporaryDirectory() as d:
        argv = [CLI, "-F", "null", "-S", mode]
        for p in paths:
            argv += ["-r", p]
        pr = subprocess.run(argv, cwd=d, capture_output=True, text=True, timeout=900)
        assert pr.returncode == 0, pr.stderr[-2000:]
        files = {}
        for n in sorted(os.listdir(d)):
            with open(os.path.join(d, n), "rb") as f:
                files[n] = f.read()
        return files, [l for l in pr.stderr.splitlines() if l.startswith("*** Saving")]


class Decoders:
    """The reference's default decoders behind r433b_dispatch_r_devices[_parallel] (state carried across files, as
    in one rtl_433 process)."""

    def __init__(self, n_sets=1):
        self.sets = [refh.Ref(chain_decoders=True, store_bitbuffers=False) for _ in range(n_sets)]
        self.n = [r.register_defaults() for r in self.sets][0]
        self.devices = self.sets[0].registered()

    def dispatch(self, ctx, n_streams):
        if len(self.sets) == 1:
            r = self.sets[0]
            ptrs = r.L.refh_begin_external_dispatch(r.h)
            try:
                for s in range(n_streams):
                    assert ctx.L.r433b_dispatch_r_devices(ctx.h, C.byref(ctx._res), s, ptrs, self.n) == 0
            finally:
                r.L.refh_end_external_dispatch(r.h)
            return
        arr = (C.c_void_p * len(self.sets))()
        for i, r in enumerate(self.sets):
            arr[i] = r.L.refh_begin_external_dispatch(r.h)
        try:
            assert ctx.L.r433b_dispatch_r_devices_parallel(ctx.h, C.byref(ctx._res), arr, self.n, len(self.sets)) == 0
        finally:
            for r in self.sets:
                r.L.refh_end_external_dispatch(r.h)

    def close(self):
        for r in self.sets:
            r.close()


def gpu_grabs(ctx, paths, mode, decoders=None, gates=False, split=None, uniform="auto", on_device=False, page=256 << 20):
    """The files the GPU path writes for `rtl_433 -S mode -r paths...` -> ({name: bytes}, stderr lines).
    split: cut the files into batches at these indices (the ring tail goes from batch to batch)."""
    ctx.set_devices(decoders.devices if decoders else lib.default_device_table())
    ctx.set_gates(lib.default_gates(decoders.devices if decoders else lib.default_device_table()) if gates else None)
    err = io.StringIO()
    bounds = [0] + list(split or []) + [len(paths)]
    with tempfile.TemporaryDirectory() as d:
        g = captures.Grabber(d, err=err, page_bytes=page)
        for lo, hi in zip(bounds[:-1], bounds[1:]):
            for batch in captures.load_batches(paths[lo:hi], uniform=uniform):
                keep = None
                data = batch["data"]
                if on_device:
                    import torch
                    keep = torch.from_numpy(data).cuda()
                    data = keep.data_ptr()
                ctx.process(data, batch["offsets"], batch["abi_format"], batch["sample_rate"], batch["center_frequency"],
                            lengths=batch["lengths"], data_on_device=on_device)
                ctx.fetch()
                if MODES[mode] != lib.GRAB_ALL:
                    decoders.dispatch(ctx, len(batch["files"]))
                if MODES[mode] == lib.GRAB_UNDECODED:
                    ctx.analyze()
                ss = {"cu8": 2, "cs8": 2, "cs16": 4, "cf32": 4}[batch["format"]]
                g.write(ctx, MODES[mode], batch["center_frequency"], batch["sample_rate"], ss)
                del keep
        files = {}
        for n in sorted(os.listdir(d)):
            with open(os.path.join(d, n), "rb") as f:
                files[n] = f.read()
    return files, [l for l in err.getvalue().splitlines() if l.startswith("*** Saving")]


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def check(case, mode, got, lines):
    """Against the compiled reference where it is built, always against the committed fingerprints."""
    assert got, (case, mode)
    want_fp = golden()[case][mode]
    assert fingerprint(got) == want_fp, (case, mode)
    if os.path.exists(CLI):
        with tempfile.TemporaryDirectory() as d:
            want, want_lines = reference_grabs(write_case(cases()[case], d), mode)
        assert sorted(want) == sorted(got), (case, mode)
        for n in want:
            assert want[n] == got[n], (case, mode, n)
        assert lines == want_lines


def modes_with_decoders(variant, mode_names=tuple(MODES)):
    """All four modes with the reference's decoders behind the dispatch: ungated, gated, or on 3 replay threads."""
    decoders = Decoders(n_sets=3 if variant == "parallel" else 1)
    ctx = lib.Context(0)
    try:
        with tempfile.TemporaryDirectory() as d:
            paths = write_case(cases()["ook_cu8"], d)
            for mode in mode_names:
                got, lines = gpu_grabs(ctx, paths, mode, decoders, gates=variant != "plain")
                check("ook_cu8", mode, got, lines)
    finally:
        ctx.close()
        decoders.close()


def formats_and_paths():
    """cs8 (grabbed as cu8), cs16, cf32 (grabbed as cs16); device input; a pipelined host batch; a run cut into two
    batches (the ring tail carried over); grab_copy in small pages."""
    ctx = lib.Context(0)
    try:
        with tempfile.TemporaryDirectory() as d:
            for case in ("ook_cs8", "fsk_cs16", "fsk_cf32"):
                os.makedirs(os.path.join(d, case))
                paths = write_case(cases()[case], os.path.join(d, case))
                got, lines = gpu_grabs(ctx, paths, "all")
                assert all(n.endswith(".cu8" if case == "ook_cs8" else ".cs16") for n in got)
                check(case, "all", got, lines)
            paths = write_case(cases()["ook_cu8"], d)
            whole, lines = gpu_grabs(ctx, paths, "all")
            check("ook_cu8", "all", whole, lines)
            assert_coverage(ctx, paths)
            assert gpu_grabs(ctx, paths, "all", split=[1, 4])[0] == whole
            assert gpu_grabs(ctx, paths, "all", page=1)[0] == whole
            assert gpu_grabs(ctx, paths, "all", uniform=True)[0] == whole
            if lib.LIB_PATH.endswith("libr433b.so"):  # real device memory
                assert gpu_grabs(ctx, paths, "all", on_device=True)[0] == whole
                assert gpu_grabs(ctx, paths[1:], "all", on_device=True)[0] == gpu_grabs(ctx, paths[1:], "all")[0]
            ctx.set_pipeline(4)
            try:
                assert gpu_grabs(ctx, paths[1:], "all", uniform=True)[0] == gpu_grabs_sequential(paths[1:])
            finally:
                ctx.set_pipeline(0)
    finally:
        ctx.close()


def assert_coverage(ctx, paths):
    """The run of `paths` (one batch) has windows that reach before the run (zeros), that start in an earlier file,
    that wrap in the ring with real bytes on both sides, that are clamped to what was pushed, and frames of packages
    from several blocks."""
    b = captures.load_batches(paths)[0]
    ctx.set_devices(lib.default_device_table())
    ctx.set_gates(None)
    ctx.process(b["data"], b["offsets"], b["abi_format"], b["sample_rate"], b["center_frequency"], lengths=b["lengths"])
    res = ctx.fetch()
    plan = ctx.grab_plan(lib.GRAB_ALL)
    cum = np.concatenate([[0], np.cumsum(b["lengths"].astype(np.int64))])
    lo = plan["run_end"] - plan["bytes"].astype(np.int64)
    wanted = (2 * plan["grab_len"].astype(np.int64) // 131072 + 1) * 131072
    blocks = [len(set(res["packages"]["block"][g["first_package"]:g["first_package"] + g["n_packages"]])) for g in plan]
    assert (lo < 0).any()
    assert (np.searchsorted(cum, lo, "right") - 1 < plan["stream"]).any()
    assert ((lo >= 0) & (lo // lib.GRAB_RING != (plan["run_end"] - 1) // lib.GRAB_RING)).any()
    assert (plan["bytes"] < wanted).any()
    assert max(blocks) > 1


def gpu_grabs_sequential(paths):
    c = lib.Context(0)
    try:
        c.set_pipeline(1)
        return gpu_grabs(c, paths, "all", uniform=True)[0]
    finally:
        c.close()


def state_errors():
    """Modes 2-4 before the dispatch, mode 4 before r433b_analyze, pulse-level batches: R433B_ESTATE."""
    ctx = lib.Context(0)
    decoders = Decoders()
    try:
        x = synth.ook_stream(7, n_samples=1 << 18, n_bursts=3)
        ctx.set_devices(decoders.devices)
        ctx.process(x, np.array([0, x.nbytes], np.uint64), lib.FMT_CU8, 250000, 433920000)
        ctx.fetch()
        assert len(ctx.grab_plan(lib.GRAB_ALL)) >= 1
        for mode in (lib.GRAB_UNKNOWN, lib.GRAB_KNOWN, lib.GRAB_UNDECODED):
            with pytest.raises(lib.R433Error, match="r433b error -5"):
                ctx.grab_plan(mode)
        decoders.dispatch(ctx, 1)
        ctx.grab_plan(lib.GRAB_UNKNOWN)
        with pytest.raises(lib.R433Error, match="r433b error -5"):
            ctx.grab_plan(lib.GRAB_UNDECODED)
        ctx.analyze()
        ctx.grab_plan(lib.GRAB_UNDECODED)
        with pytest.raises(lib.R433Error, match="r433b error -1"):
            ctx.grab_plan(5)
        p = lib.Pulses()
        pd = lib.PulseData()
        pd.sample_rate, pd.num_pulses = 250000, 3
        for i in range(3):
            pd.pulse[i], pd.gap[i] = 100, 200
        p.add(pd)
        ctx.process_pulses(p)
        ctx.fetch()
        with pytest.raises(lib.R433Error, match="r433b error -5"):
            ctx.grab_plan(lib.GRAB_ALL)
        p.close()
    finally:
        ctx.close()
        decoders.close()


def command_line_and_existing_names():
    """`python -m rtl_433_b200.captures FILES -S all --grab-dir DIR`: names that exist are skipped and the counter runs
    on, the stderr line per file is the reference's."""
    import contextlib
    with tempfile.TemporaryDirectory() as d:
        src, out = os.path.join(d, "in"), os.path.join(d, "out")
        os.makedirs(src)
        os.makedirs(out)
        paths = write_case(cases()["ook_cs8"], src)
        taken = "g002_433.92M_250k.cu8"
        open(os.path.join(out, taken), "wb").close()
        err = io.StringIO()
        with contextlib.redirect_stderr(err), contextlib.redirect_stdout(io.StringIO()):
            captures.main(paths + ["-S", "all", "--grab-dir", out])
        got = {}
        for n in sorted(os.listdir(out)):
            with open(os.path.join(out, n), "rb") as f:
                got[n] = f.read()
        assert got.pop(taken) == b""
        want = golden()["ook_cs8"]["all"]
        renamed = ["g%03d_433.92M_250k.cu8" % c for c in (1, 3, 4)]
        assert [[n, s, h] for n, (_, s, h) in zip(renamed, want)] == fingerprint(got)
        lines = [l for l in err.getvalue().splitlines() if l.startswith("*** Saving")]
        assert [l.split()[5] for l in lines] == renamed
        if os.path.exists(CLI):
            ref = os.path.join(d, "ref")
            os.makedirs(ref)
            open(os.path.join(ref, taken), "wb").close()
            pr = subprocess.run([CLI, "-F", "null", "-S", "all"] + [a for p in paths for a in ("-r", p)], cwd=ref,
                                capture_output=True, text=True, timeout=900)
            assert pr.returncode == 0
            assert sorted(os.listdir(ref)) == sorted(list(got) + [taken])
            for n in got:
                with open(os.path.join(ref, n), "rb") as f:
                    assert f.read() == got[n], n
            assert [l for l in pr.stderr.splitlines() if l.startswith("*** Saving")] == lines


needs_ref = pytest.mark.skipif(not refh.available(), reason="oracle/_ref/libr433ref.so not built (decoders)")


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("variant", ["plain", "gated", "parallel"])
def test_modes_with_reference_decoders(variant):
    modes_with_decoders(variant)


@pytest.mark.gpu
def test_formats_device_input_pipeline_prior_and_pages():
    formats_and_paths()


@pytest.mark.gpu
def test_command_line_and_existing_names():
    command_line_and_existing_names()


@pytest.mark.gpu
@needs_ref
def test_state_errors():
    state_errors()
