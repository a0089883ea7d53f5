"""-m gpu: k_front and k_detect against the oracle on hostile IQ (tests/hostile_iq.py): full-scale samples at block
starts, the rails, glitch trains, drifting noise floors, exact plateaus, pulses on every tile phase, 1200-pulse trains
and cs16 FSK at every amplitude.  Every family runs with and without stage arrays (run_gpu), at the default block
size and at block_bytes = 32768, and must equal the oracle exactly: packages, widths, every event and both stage
arrays (and the compiled reference when it is present).  Each family also asserts that it reached the path it aims
at, so that a family which stops reaching it fails.  tests/test_emu_front_fuzz.py runs the same bodies under the SIMT
emulator with fewer seeds."""
import concurrent.futures
import functools
import os
import threading

import numpy as np
import pytest

import helpers
import hostile_iq as H
import test_chain
from oracle import refh
from rtl_433_b200 import lib
from test_gpu_parity import ctx, devices, oracle_for, run_gpu  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

SEEDS = range(8)
BLOCKS = (0, 32768)


def first_difference(want, got):
    """Where two results part first: the first package whose header or widths differ, else the first stage sample."""
    for i, (p, q) in enumerate(zip(want["packages"], got["packages"])):
        if any(p[k] != q[k] for k in helpers.PKG_INT_KEYS) or not (np.array_equal(p["pulse"], q["pulse"])
                                                                  and np.array_equal(p["gap"], q["gap"])):
            return f"first differing package {i}: offset {p['offset']} (oracle) vs {q['offset']}"
    if len(want["packages"]) != len(got["packages"]):
        k = min(len(want["packages"]), len(got["packages"]))
        side, more = ("oracle", want) if len(want["packages"]) > k else ("kernels", got)
        return f"package {k} at offset {more['packages'][k]['offset']} only in the {side}"
    for s in ("am", "fm"):
        if s in want and s in got and len(want[s]) == len(got[s]) and not np.array_equal(want[s], got[s]):
            j = int(np.nonzero(want[s] != got[s])[0][0])
            return f"first differing {s} sample {j}: {want[s][max(0, j - 2):j + 4]} (oracle) vs {got[s][max(0, j - 2):j + 4]}"
    return "events differ"


def check(got, want, tag, stages=True):
    d = helpers.compare_results(want, got, tag, stages=stages)
    assert not d, f"{tag}: {first_difference(want, got)}\n" + "\n".join(d[:12])


def _groups(cases):
    """Cases that can share a batch: same format, rate, centre frequency, detector and levels."""
    out = {}
    for c in cases:
        out.setdefault((c.fmt, c.rate, c.freq, c.fpdm, tuple(sorted(c.levels.items()))), []).append(c)
    return out.values()


@functools.lru_cache(maxsize=None)
def family_cases(name, seed):
    """The cases of one family and seed, made once per process (the level fuzz runs them at many levels)."""
    return tuple(H.FAMILIES[name][0](seed))


def oracle_results(devices, cases, blocks, levels=None):
    """The oracle's result of every case at every block size, {(id(case), block_bytes): result}, on a few host threads
    (the oracle holds no global state and its calls release the interpreter lock)."""
    local = threading.local()

    def one(job):
        c, bb = job
        if not hasattr(local, "o"):
            local.o = oracle_for(devices)
            if levels:
                local.o.set_levels(**levels)
        return (id(c), bb), local.o.run(c.iq, c.fmt, c.rate, c.freq, c.fpdm, block_bytes=bb)

    with concurrent.futures.ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as ex:
        return dict(ex.map(one, [(c, bb) for c in cases for bb in blocks]))


def run_family(ctx, devices, name, seeds, blocks=BLOCKS, levels=None, evidence=True, collect=None):
    """Every case of family `name` over `seeds` through run_gpu against the oracle; the evidence checks run on the
    default levels only (magnitude mode, for one, never reaches envelope 32768).  `collect`, a list, receives
    (case, block_bytes, oracle result) of every comparison."""
    ev = H.FAMILIES[name][1]
    cases = [c for s in seeds for c in family_cases(name, s)]
    wants = oracle_results(devices, cases, blocks, levels)
    if levels:
        ctx.set_levels(**levels)
    try:
        for group in _groups(cases):
            c0 = group[0]
            for bb in blocks:
                gpu = run_gpu(ctx, [c.iq for c in group], c0.fmt, c0.rate, c0.freq, c0.fpdm, bb)
                tm = ctx.timing()
                for c, g in zip(group, gpu):
                    want = wants[(id(c), bb)]
                    check(g, want, f"{c} block_bytes {bb} levels {levels}")
                    if collect is not None:
                        collect.append((c, bb, want))
                    if evidence and not levels:
                        blk = (bb or 262144) // c.fmt
                        if name in H.TIMED:
                            ev(c, want, blk, tm)
                        else:
                            ev(c, want, blk)
    finally:
        if levels:
            ctx.set_levels()
    return cases


def against_reference(ctx, cases, levels=None):
    """The same batches against the compiled reference, where it is present (at the default levels or `levels`)."""
    if not refh.available():
        return
    r = refh.Ref(store_bitbuffers=False, store_stages=True)
    r.register_defaults()
    if levels:
        ctx.set_levels(**levels)
        r.set_levels(**levels)
    try:
        for group in _groups(cases):
            c0 = group[0]
            gpu = run_gpu(ctx, [c.iq for c in group], c0.fmt, c0.rate, c0.freq, c0.fpdm)
            for c, g in zip(group, gpu):
                check(g, r.run(c.iq, c.fmt, c.rate, c.freq, c.fpdm), f"{c} vs reference levels {levels}")
    finally:
        r.close()
        if levels:
            ctx.set_levels()


def family(ctx, devices, name, seeds):
    cases = run_family(ctx, devices, name, seeds)
    against_reference(ctx, cases[:4])


def levels(ctx, devices, seeds):
    """Magnitude mode on every family, and a fixed level on the families with full-scale samples and glitches."""
    for name in H.FAMILIES:
        run_family(ctx, devices, name, seeds, blocks=(32768,), levels=dict(use_mag_est=1))
    for name in ("spikes", "glitches"):
        run_family(ctx, devices, name, seeds, blocks=(0, 32768), levels=dict(level_limit=-8.0))


def pipelined_and_chained(ctx, devices, seeds, levels=None):
    """Full-scale spikes and glitches through the pipelined host path (time slices, state carried between launches)
    and as chained batches cut at block boundaries (state carried between calls), at the default levels or `levels`."""
    cases = [c for s in seeds for n in ("spikes", "glitches") for c in family_cases(n, s)]
    o = oracle_for(devices, stages=True)
    if levels:
        ctx.set_levels(**levels)
        o.set_levels(**levels)
    try:
        _pipelined_and_chained(ctx, cases, o)
    finally:
        if levels:
            ctx.set_levels()


def _pipelined_and_chained(ctx, cases, o):
    for bb in BLOCKS:
        wants = [o.run(c.iq, 2, block_bytes=bb) for c in cases]
        data = np.concatenate([c.iq for c in cases])
        offsets = np.concatenate([[0], np.cumsum([c.iq.nbytes for c in cases])]).astype(np.uint64)
        try:
            ctx.set_pipeline(4)
            ctx.process(data, offsets, lib.FMT_CU8, H.RATE, 433920000, lib.FPDM_AUTO, bb)
            ctx.fetch()
            assert ctx.timing()["detect_launches"] > 1
            for i, c in enumerate(cases):
                check(helpers.gpu_stream_results(ctx, i), wants[i], f"{c} pipelined block_bytes {bb}", stages=False)
        finally:
            ctx.set_pipeline(0)
        block = bb or 262144
        chunked = [test_chain.cut(c.iq, block, (1, 2, 3, 5)) for c in cases]
        got, _ = test_chain.run_chained(ctx, [[ch] for ch in chunked], lib.FMT_CU8, H.RATE, block_bytes=bb, stages=True)
        for i, c in enumerate(cases):
            g = {k: v for k, v in got[i][0].items() if k != "hdr"}
            check(g, wants[i], f"{c} chained block_bytes {bb}")


@pytest.mark.parametrize("name", list(H.FAMILIES))
def test_family(ctx, devices, name):
    family(ctx, devices, name, SEEDS)


def test_levels(ctx, devices):
    levels(ctx, devices, SEEDS[:3])


def test_pipelined_and_chained(ctx, devices):
    pipelined_and_chained(ctx, devices, SEEDS[:3])
