#!/usr/bin/env python
"""Chained batches on the BASELINE configs[1] workload (4096 x 2^20-sample cu8 streams, all 335 default devices):
one batch of whole streams against chains of 1, 2 and 4 blocks (262144 bytes each) per stream per call.

Per mode: device-resident time (IQ already on the device) and host-input time (packed pinned host chunks; packing
is not timed), both per 4.29 G samples, calls, and the chunk-end folds / FM rebuilds.  Every chained run is checked
against the one-batch run: all package headers (absolute offset, end_pos, block, seq), widths and per-(package, device)
event counts of every stream, and every event byte of 32 streams.  Prints the card and its power limit.

    python tools/chain_perf.py [--streams 4096] [--log2n 20]
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (workload generator, card identity)
import helpers  # noqa: E402
from rtl_433_b200 import lib  # noqa: E402

BLOCK = 262144
KEYS = ["seq", "type", "block", "offset", "end_pos", "start_ago", "end_ago", "num_pulses", "ook_low_estimate",
        "ook_high_estimate", "fsk_f1_est", "fsk_f2_est"]
CHECK_STREAMS = 32


class Collect:
    """Everything of a run that the comparison looks at, per stream, in (seq) order."""

    def __init__(self, n):
        self.hdr = [[] for _ in range(n)]
        self.widths = [[] for _ in range(n)]
        self.pairs = [[] for _ in range(n)]
        self.full = [helpers_empty() for _ in range(CHECK_STREAMS)]

    def add(self, ctx, res, streams):
        pk = res["packages"]
        pairs = res["pairs"]
        cols = np.stack([pk[k].astype(np.int64) for k in KEYS], 1) if len(pk) else np.zeros((0, len(KEYS)), np.int64)
        bounds = np.searchsorted(pk["stream"], np.arange(len(streams) + 1)) if len(pk) else np.zeros(len(streams) + 1, int)
        for i in range(len(streams)):
            a, b = int(bounds[i]), int(bounds[i + 1])
            if a == b:
                continue
            self.hdr[i].append(cols[a:b])
            for k in range(a, b):
                o, c = int(pk["pulse_off"][k]), int(pk["pulse_count"][k])
                self.widths[i].append(res["pulse_pool"][o:o + c].copy())
                self.widths[i].append(res["gap_pool"][o:o + c].copy())
            p = pairs[pk["first_pair"][a:b] // max(1, res["n_devices"])]  # a package's row: first_pair / n_devices
            self.pairs[i].append(np.stack([p["bytes"], p["events"], p["gated_single"], p["gated_multi"]], -1))
        for i in range(min(CHECK_STREAMS, len(streams))):
            got = helpers.gpu_stream_results(ctx, i)
            acc = self.full[i]
            k0 = len(acc["packages"])
            acc["packages"] += got["packages"]
            for e in got["events"]:
                e["package"] += k0
                acc["events"].append(e)

    def diff(self, other):
        for i in range(len(self.hdr)):
            cat = lambda xs, shape: np.concatenate(xs) if xs else np.zeros(shape, np.int64)  # noqa: E731
            if not np.array_equal(cat(self.hdr[i], (0, len(KEYS))), cat(other.hdr[i], (0, len(KEYS)))):
                return f"stream {i}: package headers differ"
            if not np.array_equal(cat(self.widths[i], 0), cat(other.widths[i], 0)):
                return f"stream {i}: widths differ"
            if not np.array_equal(cat(self.pairs[i], (0, 0, 4)), cat(other.pairs[i], (0, 0, 4))):
                return f"stream {i}: event counts differ"
        for i, (a, b) in enumerate(zip(self.full, other.full)):
            d = helpers.compare_results(a, b, f"stream {i}", stages=False)
            if d:
                return d[0]
        return None


def helpers_empty():
    return {"packages": [], "events": []}


def run(ctx, torch, dev, host, n, stride, chunk, pinned):
    """One pass over the workload in chunks of `chunk` bytes per stream (chunk == stride: one batch).
    -> (device ms, host ms, calls, folds, rebuilds, Collect of the device-resident pass)"""
    calls = stride // chunk
    coll = Collect(n)
    offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(stride)
    lens = np.full(n, chunk, np.uint64)
    dev_ms = host_ms = 0.0
    folds = rebuilds = 0
    for host_input in (False, True):
        chain = lib.Chain(ctx, n) if calls > 1 else None
        try:
            for r in range(calls):
                last = np.full(n, 1 if r == calls - 1 else 0, np.uint8)
                if host_input:
                    staged = pinned.numpy()[:n * chunk].reshape(n, chunk)
                    staged[:] = host[:, r * chunk:(r + 1) * chunk]  # packing: not timed
                    offs = np.arange(n + 1, dtype=np.uint64) * np.uint64(chunk)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ctx.process(pinned.data_ptr(), offs, lib.FMT_CU8, 250000, 433920000, lengths=lens, chain=chain,
                                last=last if chain else None)
                    ctx.fetch()
                    host_ms += (time.perf_counter() - t0) * 1e3
                else:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ctx.process(dev.data_ptr() + r * chunk, offsets, lib.FMT_CU8, 250000, 433920000, data_on_device=True,
                                lengths=lens, chain=chain, last=last if chain else None)
                    res = ctx.fetch()
                    dev_ms += (time.perf_counter() - t0) * 1e3
                    tm = ctx.timing()
                    folds += tm["chain_folds"]
                    rebuilds += tm["chain_fm_rebuilds"]
                    coll.add(ctx, res, range(n))
        finally:
            if chain:
                chain.close()
    return dev_ms, host_ms, calls, folds, rebuilds, coll


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--blocks", type=int, nargs="+", default=[1, 2, 4])
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("chain_perf: no CUDA device (there is no CPU measurement)")
    n, stride = a.streams, 2 << a.log2n
    print("card:", bench.gpu_identity(0), flush=True)
    host = np.zeros((n, stride), np.uint8)

    def sink(k, seed, x):
        host[k] = x

    bench.generate("ook", list(range(n)), 1 << a.log2n, sink)
    dev = torch.from_numpy(host.reshape(-1)).cuda()
    pinned = torch.empty(n * stride, dtype=torch.uint8).pin_memory()
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    scale = 4.29e9 / (n * (stride // 2))
    try:
        run(ctx, torch, dev, host, n, stride, stride, pinned)  # warm-up
        base = run(ctx, torch, dev, host, n, stride, stride, pinned)
        print(f"one batch: device-resident {base[0] * scale:.1f} ms, host input {base[1] * scale:.1f} ms "
              f"per 4.29 G samples", flush=True)
        for k in a.blocks:
            dm, hm, calls, folds, rebuilds, coll = run(ctx, torch, dev, host, n, stride, k * BLOCK, pinned)
            d = coll.diff(base[5])
            print(f"chained, {k} block(s) per stream per call ({calls} calls): device-resident {dm * scale:.1f} ms "
                  f"({dm / calls:.2f} ms per call), host input {hm * scale:.1f} ms, chunk-end folds {folds}, "
                  f"FM rebuilds {rebuilds}, {'equal to the one-batch run' if d is None else 'DIFFERS: ' + d}",
                  flush=True)
            if d is not None:
                sys.exit(1)
    finally:
        ctx.close()


if __name__ == "__main__":
    main()
