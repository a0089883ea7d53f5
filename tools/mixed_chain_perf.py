"""Mixed chained batches (r433b_process_mixed_chained) against one chain per (format, rate, frequency) group,
device-resident.

The corpus is that of tools/mixed_perf.py: four classes, 1,792 files of 2^20 samples (cu8 250k OOK x 1024, cs16 1024k
FSK x 256, cu8 1024k FSK x 256, cs8 250k OOK x 256), fed chunk by chunk, K blocks of the file's own input per call
(262144 bytes a block).  The grouped way keeps four one-format chains (r433b_process_chained) and calls them one after
another every round; the mixed way keeps one chain of 1,792 slots and makes one call per round.  With the reference's
335 default devices, the two alternate in one process at K = 1, 2 and 4.  Per way and K it prints the wall time per
round (process and fetch, a round's calls summed), the k_detect span per round, k_mixed_order's time, and whether every
slot's package count, event count and digest of every round are equal.  Output: one JSON line per pass, then a summary
line with the card and its power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rtl_433_b200 import lib  # noqa: E402
from mixed_perf import card, classes  # noqa: E402

BLOCK = 262144


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--log2-samples", type=int, default=20)
    ap.add_argument("--scale", type=int, default=1, help="divide every class's file count by this")
    ap.add_argument("--distinct", type=int, default=4)
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--blocks", default="1,2,4", help="blocks per call")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mixed_chain_perf: no CUDA device (there is no CPU path)")
    cls = classes(1 << a.log2_samples, a.scale, a.distinct)
    # one device buffer: the classes back to back, files on a uniform stride within each
    parts, groups = [], []
    at = 0
    for tag, fmt, rate, freq, count, files in cls:
        stride = (max(len(f) for f in files) + 31) // 32 * 32
        host = np.zeros(stride * count, np.uint8)
        lens = np.zeros(count, np.uint64)
        for i in range(count):
            f = files[i % len(files)]
            host[i * stride:i * stride + len(f)] = f
            lens[i] = len(f)
        groups.append({"tag": tag, "fmt": fmt, "rate": rate, "freq": freq, "count": count,
                       "off": at + np.arange(count, dtype=np.uint64) * np.uint64(stride), "len": lens})
        parts.append(host)
        at += len(host)
    dev = torch.from_numpy(np.concatenate(parts)).cuda()
    base = dev.data_ptr()
    n_all = sum(g["count"] for g in groups)
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())

    def chunk(g, r, k):
        """Round r's chunks of group g at k blocks per call -> offsets (n + 1), lengths, last, whether any is live."""
        step = np.uint64(k * BLOCK)
        done = np.minimum(g["len"], np.uint64(r) * step)
        lens = np.minimum(g["len"] - done, step)
        offs = np.append(g["off"] + done, g["off"][-1] + done[-1] + step).astype(np.uint64)
        last = (done + lens >= g["len"]).astype(np.uint8)
        return offs, lens, last, bool((done < g["len"]).any()) or r == 0

    def rounds(k):
        return max(int(-(-int(g["len"].max()) // (k * BLOCK))) for g in groups)

    def grouped(k):
        walls, detect, out = [], [], []
        chains = [lib.Chain(ctx, g["count"]) for g in groups]
        try:
            for r in range(rounds(k)):
                w = d = 0.0
                row = []
                for g, ch in zip(groups, chains):
                    offs, lens, last, live = chunk(g, r, k)
                    if not live:
                        row += [(0, 0, 0)] * g["count"]
                        continue
                    t0 = time.perf_counter()
                    ctx.process(base, offs, g["fmt"], g["rate"], g["freq"], data_on_device=True, lengths=lens,
                                chain=ch, last=last)
                    res = ctx.fetch()
                    w += time.perf_counter() - t0
                    d += ctx.timing()["detect_ms"]
                    row += per_slot(res, g["count"])
                walls.append(w)
                detect.append(d)
                out.append(row)
        finally:
            for ch in chains:
                ch.close()
        return walls, detect, [0.0] * len(walls), out

    def per_slot(res, n):
        pk = res["packages"]
        counts = np.bincount(pk["stream"], minlength=n) if len(pk) else np.zeros(n, np.int64)
        return [(int(counts[s]), 0, ctx.stream_digest(s)) for s in range(n)]

    def mixed(k):
        walls, detect, order, out = [], [], [], []
        fmts = [g["fmt"] for g in groups for _ in range(g["count"])]
        rates = [g["rate"] for g in groups for _ in range(g["count"])]
        freqs = [g["freq"] for g in groups for _ in range(g["count"])]
        with lib.Chain(ctx, n_all) as ch:
            for r in range(rounds(k)):
                cs = [chunk(g, r, k) for g in groups]
                offs = np.concatenate([c[0][:-1] for c in cs] + [[at]]).astype(np.uint64)
                lens = np.concatenate([c[1] for c in cs]).astype(np.uint64)
                last = np.concatenate([c[2] for c in cs]).astype(np.uint8)
                t0 = time.perf_counter()
                ctx.process_mixed(base, offs, fmts, rates, freqs, lengths=lens, data_on_device=True, chain=ch, last=last)
                res = ctx.fetch()
                walls.append(time.perf_counter() - t0)
                tm = ctx.timing()
                detect.append(tm["detect_ms"])
                order.append(tm["mixed_order_ms"])
                row = per_slot(res, n_all)
                # a group whose files have all ended makes no call in the grouped way
                lo = 0
                for g, c in zip(groups, cs):
                    if not c[3]:
                        row[lo:lo + g["count"]] = [(0, 0, 0)] * g["count"]
                    lo += g["count"]
                out.append(row)
        return walls, detect, order, out

    ks = [int(x) for x in a.blocks.split(",")]
    for k in ks:  # warm-up of both ways at every chunk size
        grouped(k)
        mixed(k)
    rows = []
    for p in range(a.passes):
        for k in ks:
            gw, gd, _, go = grouped(k)
            mw, md, mo, mo_out = mixed(k)
            row = {"pass": p, "blocks_per_call": k, "rounds": len(gw),
                   "grouped_ms_per_round": round(1e3 * sum(gw) / len(gw), 2),
                   "mixed_ms_per_round": round(1e3 * sum(mw) / len(mw), 2),
                   "grouped_detect_ms_per_round": round(sum(gd) / len(gd), 2),
                   "mixed_detect_ms_per_round": round(sum(md) / len(md), 2),
                   "mixed_order_ms_per_round": round(sum(mo) / len(mo), 3),
                   "equal": go == mo_out}
            rows.append(row)
            print(json.dumps(row), flush=True)
    ctx.close()
    summary = {"card": card(), "slots": n_all, "samples_per_file": 1 << a.log2_samples,
               "all_equal": all(r["equal"] for r in rows)}
    for k in ks:
        summary[f"k{k}"] = {w: min(r[f"{w}_ms_per_round"] for r in rows if r["blocks_per_call"] == k)
                            for w in ("grouped", "mixed")}
    print(json.dumps(summary))
    if not summary["all_equal"]:
        raise SystemExit("mixed_chain_perf: results differ")


if __name__ == "__main__":
    main()
