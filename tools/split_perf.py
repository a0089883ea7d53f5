#!/usr/bin/env python
"""Segmented replay (r433b_set_split) against the one-warp walk, on the workloads it is for and on the one it is not.

  (a) one cu8 250 kS/s OOK stream of 2^30 samples (about 72 minutes), seeded synth.ook_stream pieces of 2^20 samples
      with bursts throughout;
  (b) one cs16 1.024 MS/s 2-FSK stream of 2^28 samples (synth.fsk_stream pieces, FM on);
  (c) 16 cu8 streams of 2^27 samples (as (a));
  (d) BASELINE configs[1]: 4096 cu8 streams of 2^20 samples, with R433B_SPLIT_AUTO, which must not split it.

Every workload is device-resident (no copy-in), all 335 default devices, the reference's 262144-byte blocks.  Each
runs once untimed per mode (buffer growth), then `--repeats` times unsplit and split (R433B_SPLIT_AUTO) alternating.
Per call: total time (host clock around r433b_process + r433b_fetch, synchronous), front_ms, detect_ms, slice_ms,
split_merge_ms, segments / rewalks / rounds, and whether the outputs are the same: package count, event count and bytes,
and every stream's r433b_stream_digest (package headers, widths and every event).  The merge's bytes moved are counted
from the merged arrays: every kept package header read and written once, every kept pulse and gap width read and
written once (the headers of discarded walks, also read, are not counted: a lower bound).  Prints the card and its
power limit.  JSON lines go to stdout.

    python tools/split_perf.py [--repeats 3] [--only a b c d]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generator, card identity)
from rtl_433_b200 import lib  # noqa: E402

PIECE = 1 << 20


def workload(name):
    """-> (host uint8 data, offsets, format, rate, frequency, fpdm)"""
    if name == "d":
        n_streams, per, kind = 4096, 1, "ook"
    elif name == "c":
        n_streams, per, kind = 16, 128, "ook"
    elif name == "b":
        n_streams, per, kind = 1, 256, "fsk"
    else:
        n_streams, per, kind = 1, 1024, "ook"
    ss = 4 if kind == "fsk" else 2
    stride = per * PIECE * ss
    host = np.empty(n_streams * stride, np.uint8)

    def sink(k, seed, x):
        host[k * PIECE * ss:(k + 1) * PIECE * ss] = x.view(np.uint8).ravel()

    bench.generate(kind, list(range(10000, 10000 + n_streams * per)), PIECE, sink)
    offsets = np.arange(n_streams + 1, dtype=np.uint64) * np.uint64(stride)
    if kind == "fsk":
        return host, offsets, lib.FMT_CS16, 1024000, 868000000, lib.FPDM_MINMAX
    return host, offsets, lib.FMT_CU8, 250000, 433920000, lib.FPDM_AUTO


def call(ctx, torch, dev, offsets, fmt, rate, freq, fpdm, split):
    ctx.set_split(split)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ctx.process(dev.data_ptr(), offsets, fmt, rate, freq, fpdm, data_on_device=True)
    res = ctx.fetch()
    wall = (time.perf_counter() - t0) * 1e3
    tm = ctx.timing()
    n_streams = len(offsets) - 1
    out = {"total_ms": round(wall, 3)}
    for k in ("front_ms", "detect_ms", "slice_ms", "split_merge_ms"):
        out[k] = round(tm[k], 3)
    for k in ("detect_launches", "split_segments", "split_rewalks", "split_rounds"):
        out[k] = tm[k]
    pk = res["packages"]
    if split and tm["split_segments"]:
        kept_pool = int(pk["pulse_count"].astype(np.int64).sum())
        moved = 2 * len(pk) * 72 + 4 * kept_pool * 4
        out["merge_bytes"] = moved
        out["merge_gbs"] = round(moved / (tm["split_merge_ms"] * 1e-3) / 1e9, 1) if tm["split_merge_ms"] else None
    digest = [ctx.stream_digest(i) for i in range(n_streams)]
    return out, (int(res["n_packages"]), int(res["n_events"]), int(res["event_bytes"]), tuple(digest))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", nargs="*", default=["a", "b", "c", "d"])
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("split_perf: no CUDA device (there is no CPU path)")
    print(json.dumps({"card": bench.gpu_identity(0), "library": lib.LIB_PATH}), flush=True)
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    try:
        for name in a.only:
            host, offsets, fmt, rate, freq, fpdm = workload(name)
            dev = torch.from_numpy(host).cuda()
            del host
            outputs = {}
            for split in (0, lib.SPLIT_AUTO):  # untimed: buffer growth
                call(ctx, torch, dev, offsets, fmt, rate, freq, fpdm, split)
            for rep in range(a.repeats):
                for split in (0, lib.SPLIT_AUTO):
                    row, outp = call(ctx, torch, dev, offsets, fmt, rate, freq, fpdm, split)
                    outputs.setdefault(split, outp)
                    row.update({"workload": name, "mode": "split" if split else "unsplit", "rep": rep,
                                "same_as_unsplit": outp == outputs[0] if 0 in outputs else None})
                    print(json.dumps(row), flush=True)
            del dev
            torch.cuda.empty_cache()
    finally:
        ctx.close()


if __name__ == "__main__":
    main()
