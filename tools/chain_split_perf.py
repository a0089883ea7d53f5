#!/usr/bin/env python
"""Segmented replay on chained batches (r433b_chain_split) against the one-warp walk of each chunk, on a recording fed
through a one-slot chain in whole-block chunks, as a recording too large for the device would be.

  (a) one cu8 250 kS/s OOK stream of 2^30 samples (about 72 minutes), seeded synth.ook_stream pieces of 2^20 samples
      with bursts throughout (as tools/split_perf.py (a));
  (b) one cs16 1.024 MS/s 2-FSK stream of 2^28 samples (synth.fsk_stream pieces, FM on).

The stream is device-resident (each chunk is a view into it, no copy-in), all 335 default devices, the reference's
262144-byte blocks.  Each chunk size runs the whole stream once untimed per mode (buffer growth), then `--repeats`
times unsplit and split (R433B_SPLIT_AUTO) alternating.  Per run: ms per call (host clock around r433b_process_chained
+ r433b_fetch, synchronous) and in total, detect_ms summed, segments / rewalks / rounds summed over the calls, and
whether the outputs are the same as the unsplit run's: every call's package count, event count and bytes, and stream
digest (package headers, widths and every event).  Prints the card and its power limit.  JSON lines go to stdout.

    python tools/chain_split_perf.py [--repeats 2] [--only a b] [--chunks 26 28]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (card identity)
import split_perf  # noqa: E402  (workloads)
from rtl_433_b200 import lib  # noqa: E402

BLOCK = 262144


def run(ctx, torch, dev, n_bytes, chunk_bytes, fmt, rate, freq, fpdm, split):
    """The whole stream through a fresh one-slot chain, chunk by chunk -> (row, outputs per call)."""
    calls, outputs = [], []
    sums = {k: 0 for k in ("detect_launches", "split_segments", "split_rewalks", "split_rounds")}
    detect_ms = 0.0
    with lib.Chain(ctx, 1) as chain:
        chain.split(split)
        torch.cuda.synchronize()
        t_all = time.perf_counter()
        for lo in range(0, n_bytes, chunk_bytes):
            n = min(chunk_bytes, n_bytes - lo)
            t0 = time.perf_counter()
            ctx.process(dev.data_ptr() + lo, [0, n], fmt, rate, freq, fpdm, BLOCK, data_on_device=True, chain=chain,
                        last=[int(lo + n >= n_bytes)])
            res = ctx.fetch()
            calls.append((time.perf_counter() - t0) * 1e3)
            tm = ctx.timing()
            detect_ms += tm["detect_ms"]
            for k in sums:
                sums[k] += tm[k]
            outputs.append((int(res["n_packages"]), int(res["n_events"]), int(res["event_bytes"]), ctx.stream_digest(0)))
        total = (time.perf_counter() - t_all) * 1e3
    row = {"calls": len(calls), "total_ms": round(total, 1), "ms_per_call": round(float(np.mean(calls)), 1),
           "max_call_ms": round(max(calls), 1), "detect_ms": round(detect_ms, 1), **sums,
           "packages": sum(o[0] for o in outputs), "events": sum(o[1] for o in outputs)}
    return row, outputs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--only", nargs="*", default=["a", "b"])
    ap.add_argument("--chunks", nargs="*", type=int, default=[26, 28], help="log2 of the samples per chunk")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("chain_split_perf: no CUDA device (there is no CPU path)")
    print(json.dumps({"card": bench.gpu_identity(0), "library": lib.LIB_PATH}), flush=True)
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    try:
        for name in a.only:
            host, offsets, fmt, rate, freq, fpdm = split_perf.workload(name)
            dev = torch.from_numpy(host).cuda()
            n_bytes = int(offsets[-1])
            ss = 4 if fmt == lib.FMT_CS16 else 2
            del host
            for log2 in a.chunks:
                chunk_bytes = (1 << log2) * ss
                assert chunk_bytes % BLOCK == 0
                for split in (0, lib.SPLIT_AUTO):  # untimed: buffer growth
                    run(ctx, torch, dev, n_bytes, chunk_bytes, fmt, rate, freq, fpdm, split)
                unsplit = None
                for rep in range(a.repeats):
                    for split in (0, lib.SPLIT_AUTO):
                        row, outp = run(ctx, torch, dev, n_bytes, chunk_bytes, fmt, rate, freq, fpdm, split)
                        if not split:
                            unsplit = unsplit or outp
                        row.update({"workload": name, "chunk_samples": 1 << log2, "mode": "split" if split else "unsplit",
                                    "rep": rep, "same_as_unsplit": outp == unsplit})
                        print(json.dumps(row), flush=True)
            del dev
            torch.cuda.empty_cache()
    finally:
        ctx.close()


if __name__ == "__main__":
    main()
