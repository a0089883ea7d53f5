#!/usr/bin/env python
"""The signal grabber on chains (r433b_chain_grab), BASELINE configs[1] workload (4096 x 2^20-sample cu8 streams, all
335 default devices), device-resident, at 1, 2 and 4 blocks (262144 bytes) per stream per call.

Per cadence: the chained run without grabbing, then with `-S all` (mode 1): time per call (host clock around
process + fetch [+ plan + copy], each call synchronous), and the device time per call of
- k_grab_ring (r433b_timing.grab_ring_ms; with chunks over one block it includes the k_grab that saves the ring bytes
  the append overwrites), which moves 2 x (appended + saved) bytes, and
- k_grab (grab_ms of the copy), which moves 2 x the bytes gathered,
each as bytes per second against the 3.35 TB/s HBM3 data-sheet peak.  Prints the card and its power limit.

    python tools/chain_grab_perf.py [--streams 4096] [--log2n 20] [--blocks 1 2 4] [--repeats 2] [--no-grab]

Every cadence runs once untimed first (buffer growth), then `--repeats` timed passes of each kind, alternating.
--no-grab times the chained runs alone (also on a build without grabbing on chains, for a comparison).
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generator, card identity)
from rtl_433_b200 import lib  # noqa: E402

BLOCK = 262144
HBM = 3.35e12


def saved_bytes(n, chunk, call):
    """Ring bytes the append of call `call` overwrites that its frames may still read (r433b_api.cu)."""
    S = lib.GRAB_RING
    c0, c1 = call * chunk, (call + 1) * chunk
    return n * max(0, min(c0, c1 - S) - max(0, c0 + min(BLOCK, chunk) - S))


def run(ctx, torch, dev, n, stride, chunk, grab):
    """One device-resident pass in chunks of `chunk` bytes per stream -> dict of totals."""
    calls = stride // chunk
    offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(stride)
    lens = np.full(n, chunk, np.uint64)
    t = {"calls": calls, "wall_ms": 0.0, "ring_ms": 0.0, "ring_bytes": 0, "grab_ms": 0.0, "grab_bytes": 0, "grabs": 0}
    with lib.Chain(ctx, n) as chain:
        if grab:
            chain.grab(lib.GRAB_ALL)
        for r in range(calls):
            last = np.full(n, 1 if r == calls - 1 else 0, np.uint8)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.process(dev.data_ptr() + r * chunk, offsets, lib.FMT_CU8, 250000, 433920000, data_on_device=True,
                        lengths=lens, chain=chain, last=last)
            ctx.fetch()
            if grab:
                ring_ms = ctx.timing()["grab_ring_ms"]
                plan = ctx.grab_plan(lib.GRAB_ALL)
                total = int(plan["bytes"].sum())
                if len(plan):
                    ctx.grab_copy(0, len(plan), total)
                    t["grab_ms"] += ctx.timing()["grab_ms"]
                t["ring_ms"] += ring_ms
                t["ring_bytes"] += 2 * (n * min(chunk, lib.GRAB_RING) + saved_bytes(n, chunk, r))
                t["grab_bytes"] += 2 * total
                t["grabs"] += len(plan)
            t["wall_ms"] += (time.perf_counter() - t0) * 1e3
    return t


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--blocks", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-grab", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("chain_grab_perf: no CUDA device (there is no CPU measurement)")
    n, stride = a.streams, 2 << a.log2n
    print("card:", bench.gpu_identity(0), "library:", lib.LIB_PATH, flush=True)
    host = np.zeros((n, stride), np.uint8)

    def sink(k, seed, x):
        host[k] = x

    bench.generate("ook", list(range(n)), 1 << a.log2n, sink)
    dev = torch.from_numpy(host.reshape(-1)).cuda()
    del host
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    try:
        kinds = (False,) if a.no_grab else (False, True)
        for k in a.blocks:
            for grab in kinds:
                run(ctx, torch, dev, n, stride, k * BLOCK, grab)  # warm-up
            for grab in [g for _ in range(a.repeats) for g in kinds]:
                t = run(ctx, torch, dev, n, stride, k * BLOCK, grab)
                c = t["calls"]
                line = f"{k} block(s) per call, {'grab mode 1' if grab else 'no grabbing'}: {c} calls, " \
                       f"{t['wall_ms'] / c:.2f} ms per call"
                if grab:
                    ring = t["ring_bytes"] / (t["ring_ms"] / 1e3) if t["ring_ms"] else 0.0
                    gat = t["grab_bytes"] / (t["grab_ms"] / 1e3) if t["grab_ms"] else 0.0
                    line += (f"; k_grab_ring {t['ring_ms'] / c:.3f} ms per call, {t['ring_bytes'] / c / 1e9:.3f} GB moved, "
                             f"{ring / 1e9:.0f} GB/s = {100 * ring / HBM:.0f} % of HBM peak; k_grab {t['grab_ms'] / c:.3f} ms "
                             f"per call, {t['grab_bytes'] / c / 1e9:.3f} GB moved, {gat / 1e9:.0f} GB/s = "
                             f"{100 * gat / HBM:.0f} % of HBM peak; {t['grabs']} grabs")
                print(line, flush=True)
    finally:
        ctx.close()


if __name__ == "__main__":
    main()
