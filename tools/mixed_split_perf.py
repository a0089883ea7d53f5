"""Segmented replay of mixed batches (r433b_process_mixed under r433b_set_split(SPLIT_AUTO)), device-resident.

(a) A few long files, one per class: cu8 250k OOK at 433.92 MHz (2^28 samples), cs8 250k at 315 MHz (2^28), cs16 1024k
    FSK at 868 MHz (2^27) and cf32 1024k FSK at 915 MHz (2^26).  Three modes: the mixed batch unsplit, the mixed batch
    split, and one r433b_process() per group with SPLIT_AUTO (times summed).
(b) The 1,792-file corpus of tools/mixed_perf.py: the mixed batch unsplit against SPLIT_AUTO.
Each file is a few distinct synthesised pieces tiled to its length.  With the reference's 335 default devices and
262144-byte blocks, the modes alternate in one process, --passes passes each after one warm-up pass.  Per pass it prints
the wall time (process and fetch; the digests are left out), detect_ms, the split counters, and whether every stream's
package count and digest and the event totals equal the first mode's.  Output: one JSON line per (case, pass, mode),
then a summary line with the card and its power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mixed_perf  # noqa: E402
from rtl_433_b200 import lib, synth  # noqa: E402


def tiled(piece, total_bytes):
    return np.resize(piece.view(np.uint8).ravel(), total_bytes)


def long_files(log2_piece):
    p = 1 << log2_piece
    ook = synth.ook_stream(11, n_samples=p, n_bursts=8, rate=250000)
    cs8 = synth.ook_stream(12, n_samples=p, n_bursts=8, rate=250000) ^ 0x80
    fsk = synth.fsk_stream(13, n_samples=p, n_bursts=4, rate=1024000)
    cf32 = (synth.fsk_stream(14, n_samples=p, n_bursts=4, rate=1024000).astype(np.float32) / np.float32(32767.0))
    return [("cu8_250k_433.92M", tiled(ook, 2 << 28), lib.FMT_CU8, 250000, 433920000),
            ("cs8_250k_315M", tiled(cs8, 2 << 28), lib.FMT_CS8, 250000, 315000000),
            ("cs16_1024k_868M", tiled(fsk, 4 << 27), lib.FMT_CS16, 1024000, 868000000),
            ("cf32_1024k_915M", tiled(cf32, 8 << 26), lib.FMT_CF32, 1024000, 915000000)]


def corpus_files(log2_samples):
    out = []
    for tag, fmt, rate, freq, count, files in mixed_perf.classes(1 << log2_samples, 1, 4):
        out += [(tag, files[i % len(files)].view(np.uint8).ravel(), fmt, rate, freq) for i in range(count)]
    return out


def upload(files, torch):
    offsets, at = [], 0
    for f in files:
        offsets.append(at)
        at += (len(f[1]) + 31) // 32 * 32
    offsets.append(at)
    host = np.zeros(at, np.uint8)
    for f, o in zip(files, offsets):
        host[o:o + len(f[1])] = f[1]
    return torch.from_numpy(host).cuda(), np.array(offsets, np.uint64)


def result(ctx, res, n):
    per_stream = np.bincount(res["packages"]["stream"].astype(np.int64), minlength=n).tolist()
    return per_stream, res["n_events"], [ctx.stream_digest(i) for i in range(n)]


def run_mixed(ctx, files, base, offsets, split):
    ctx.set_split(split)
    try:
        t0 = time.perf_counter()
        ctx.process_mixed(base, offsets, [f[2] for f in files], [f[3] for f in files], [f[4] for f in files],
                          data_on_device=True)
        res = ctx.fetch()
        wall = time.perf_counter() - t0
    finally:
        ctx.set_split(0)
    return wall, ctx.timing(), result(ctx, res, len(files))


def run_grouped(ctx, files, base, offsets):
    """One r433b_process() per (format, rate, frequency) group, SPLIT_AUTO; the streams keep the batch's order."""
    groups = {}
    for i, f in enumerate(files):
        groups.setdefault((f[2], f[3], f[4]), []).append(i)
    wall, tot = 0.0, {"detect_ms": 0.0, "split_segments": 0, "split_rewalks": 0, "split_rounds": 0}
    per_stream, events, digests = [0] * len(files), 0, [0] * len(files)
    ctx.set_split(lib.SPLIT_AUTO)
    try:
        for (fmt, rate, freq), idx in groups.items():
            # a group's files lie back to back in the buffer
            offs = np.array([int(offsets[i]) for i in idx] + [int(offsets[idx[-1] + 1])], np.uint64)
            lens = [len(files[i][1]) for i in idx]
            t0 = time.perf_counter()
            ctx.process(base + int(offs[0]), offs - offs[0], fmt, rate, freq, data_on_device=True, lengths=lens)
            res = ctx.fetch()
            wall += time.perf_counter() - t0
            tm = ctx.timing()
            for k in tot:
                tot[k] += tm[k]
            ps, ev, dg = result(ctx, res, len(idx))
            events += ev
            for j, i in enumerate(idx):
                per_stream[i], digests[i] = ps[j], dg[j]
    finally:
        ctx.set_split(0)
    return wall, tot, (per_stream, events, digests)


def case(ctx, name, files, modes, passes, torch):
    dev, offsets = upload(files, torch)
    base = dev.data_ptr()
    fns = {"unsplit": lambda: run_mixed(ctx, files, base, offsets, 0),
           "split": lambda: run_mixed(ctx, files, base, offsets, lib.SPLIT_AUTO),
           "grouped_split": lambda: run_grouped(ctx, files, base, offsets)}
    for m in modes:  # warm-up
        fns[m]()
    rows, first = [], None
    for p in range(passes):
        for m in modes:
            wall, tm, out = fns[m]()
            first = first or out
            row = {"case": name, "pass": p, "mode": m, "wall_s": round(wall, 4), "detect_ms": round(tm["detect_ms"], 2),
                   "segments": tm["split_segments"], "rewalks": tm["split_rewalks"], "rounds": tm["split_rounds"],
                   "packages": sum(out[0]), "events": out[1],
                   "equal": out[0] == first[0] and out[1] == first[1] and out[2] == first[2]}
            if "detect_launches" in tm:
                row["detect_launches"] = tm["detect_launches"]
            rows.append(row)
            print(json.dumps(row), flush=True)
    del dev
    return {m: min(r["wall_s"] for r in rows if r["mode"] == m) for m in modes}, all(r["equal"] for r in rows)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--log2-piece", type=int, default=22, help="samples of each distinct piece the long files tile")
    ap.add_argument("--log2-samples", type=int, default=20, help="samples per file of the (b) corpus")
    ap.add_argument("--cases", default="a,b")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mixed_split_perf: no CUDA device (there is no CPU path)")
    card = mixed_perf.card()  # name and power limit, read in the same call as the measurement
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    summary = {"card": card}
    if "a" in a.cases:
        summary["a_min_wall_s"], summary["a_equal"] = case(ctx, "a", long_files(a.log2_piece),
                                                           ("unsplit", "split", "grouped_split"), a.passes, torch)
    if "b" in a.cases:
        summary["b_min_wall_s"], summary["b_equal"] = case(ctx, "b", corpus_files(a.log2_samples), ("unsplit", "split"),
                                                           a.passes, torch)
    ctx.close()
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
