"""Mixed batches (r433b_process_mixed) against one batch per (format, rate, frequency) group, device-resident.

The corpus has four classes (sizes in samples per file, 2^20 by default):
  A  cu8 250k at 433.92 MHz (OOK)      x 1024
  B  cs16 1024k at 868 MHz (FSK, FM on) x 256
  C  cu8 1024k at 868 MHz (FSK)         x 256
  D  cs8 250k at 315 MHz (OOK)          x 256
A few distinct files per class are synthesised and tiled.  With the reference's 335 default devices, passes alternate
between the grouped path (four r433b_process() calls, times summed) and one mixed batch, in one process.  Per pass it
prints the wall time (process and fetch; the digests are left out), the kernel sums, k_mixed_order's time, and
whether the package and event counts and every stream's digest are equal.  Output: one JSON line per pass, then a
summary line with the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rtl_433_b200 import lib, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def classes(n, scale, distinct):
    def ook(seed, rate):
        return synth.ook_stream(seed, n_samples=n, n_bursts=8, rate=rate)
    return [("A", lib.FMT_CU8, 250000, 433920000, 1024 // scale, [ook(100 + i, 250000) for i in range(distinct)]),
            ("B", lib.FMT_CS16, 1024000, 868000000, 256 // scale,
             [synth.fsk_stream(200 + i, n_samples=n, n_bursts=4, rate=1024000).view(np.uint8) for i in range(distinct)]),
            ("C", lib.FMT_CU8, 1024000, 868000000, 256 // scale,
             [synth.fsk_burst_stream(300 + i, 96, n_samples=n, rate=1024000, cu8=True, alternate=False) for i in range(distinct)]),
            ("D", lib.FMT_CS8, 250000, 315000000, 256 // scale, [ook(400 + i, 250000) ^ 0x80 for i in range(distinct)])]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--log2-samples", type=int, default=20)
    ap.add_argument("--scale", type=int, default=1, help="divide every class's file count by this")
    ap.add_argument("--distinct", type=int, default=4)
    ap.add_argument("--passes", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mixed_perf: no CUDA device (there is no CPU path)")
    cls = classes(1 << a.log2_samples, a.scale, a.distinct)
    # one device buffer: the classes back to back, files on a uniform stride within each
    parts, groups, fmts, rates, freqs, offsets = [], [], [], [], [], []
    at = 0
    for tag, fmt, rate, freq, count, files in cls:
        stride = max(len(f) for f in files)
        stride = (stride + 31) // 32 * 32
        host = np.zeros(stride * count, np.uint8)
        for i in range(count):
            f = files[i % len(files)]
            host[i * stride:i * stride + len(f)] = f
        groups.append((tag, fmt, rate, freq, at, stride, count))
        for i in range(count):
            offsets.append(at + i * stride)
            fmts.append(fmt)
            rates.append(rate)
            freqs.append(freq)
        parts.append(host)
        at += len(host)
    offsets.append(at)
    dev = torch.from_numpy(np.concatenate(parts)).cuda()
    base = dev.data_ptr()
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())

    def grouped():
        t0 = time.perf_counter()
        sums = {"front_ms": 0.0, "detect_ms": 0.0, "slice_ms": 0.0}
        pk = ev = 0
        digests = []
        for tag, fmt, rate, freq, off, stride, count in groups:
            ctx.process(base + off, np.arange(count + 1, dtype=np.uint64) * np.uint64(stride), fmt, rate, freq,
                        data_on_device=True)
            res = ctx.fetch()
            tm = ctx.timing()
            for k in sums:
                sums[k] += tm[k]
            pk += res["n_packages"]
            ev += res["n_events"]
            t1 = time.perf_counter()
            digests += [ctx.stream_digest(i) for i in range(count)]  # outside the timed region
            t0 += time.perf_counter() - t1
        return time.perf_counter() - t0, sums, pk, ev, digests

    def mixed():
        t0 = time.perf_counter()
        ctx.process_mixed(base, np.array(offsets, np.uint64), fmts, rates, freqs, data_on_device=True)
        res = ctx.fetch()
        wall = time.perf_counter() - t0
        tm = ctx.timing()
        digests = [ctx.stream_digest(i) for i in range(len(fmts))]
        return wall, tm, res["n_packages"], res["n_events"], digests

    grouped()  # warm-up of both paths
    mixed()
    rows = []
    for p in range(a.passes):
        gw, gs, gpk, gev, gd = grouped()
        mw, mt, mpk, mev, md = mixed()
        row = {"pass": p, "grouped_s": round(gw, 4), "mixed_s": round(mw, 4),
               "grouped_kernels_ms": {k: round(v, 2) for k, v in gs.items()},
               "mixed_kernels_ms": {k: round(mt[k], 2) for k in ("front_ms", "detect_ms", "slice_ms")},
               "mixed_order_ms": round(mt["mixed_order_ms"], 3), "mixed_classes": mt["mixed_classes"],
               "packages_equal": gpk == mpk, "events_equal": gev == mev, "digests_equal": gd == md,
               "packages": mpk, "events": mev}
        rows.append(row)
        print(json.dumps(row), flush=True)
    ctx.close()
    print(json.dumps({"card": card(), "streams": len(fmts), "samples_per_file": 1 << a.log2_samples,
                      "grouped_s_min": min(r["grouped_s"] for r in rows), "mixed_s_min": min(r["mixed_s"] for r in rows),
                      "all_equal": all(r["packages_equal"] and r["events_equal"] and r["digests_equal"] for r in rows)}))


if __name__ == "__main__":
    main()
