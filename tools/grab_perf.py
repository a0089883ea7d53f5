"""k_grab throughput: `-S all` on the BASELINE configs[1] batch (4096 x 2^20-sample 250 kS/s cu8 streams, bench.py's
generator and seeds 0..N-1).  The batch is processed and fetched once; then every file of the grab plan is gathered
in pages by r433b_grab_copy(), `--repeats` times.  k_grab's time is the CUDA-event time the library records around
each launch (r433b_timing.grab_ms); the copy to the host is not in it.  Bytes moved are 2 x the bytes gathered (one
read of the batch, one write of the staging buffer).  Prints one JSON line with the card's name and power limit,
read in the same run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_HBM = 3.35e12  # H100 SXM data sheet, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, limit = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")[:2]
    return name, limit


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--page-mib", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bench
    from rtl_433_b200 import lib
    n = 1 << a.log2n
    stride = 2 * n
    data = np.empty(a.streams * stride, np.uint8)

    def sink(k, _seed, x):
        data[k * stride:(k + 1) * stride] = x
    bench.generate("ook", list(range(a.streams)), n, sink)
    offs = np.arange(a.streams + 1, dtype=np.uint64) * np.uint64(stride)
    ctx = lib.Context(0)
    ctx.set_devices(lib.default_device_table())
    ctx.process(data, offs, lib.FMT_CU8, 250000, 433920000)
    res = ctx.fetch()
    plan = ctx.grab_plan(lib.GRAB_ALL)
    sizes = plan["bytes"].astype(np.int64)
    pages, i, page = [], 0, a.page_mib << 20
    while i < len(plan):
        j, tot = i, 0
        while j < len(plan) and (j == i or tot + int(sizes[j]) <= page):
            tot += int(sizes[j])
            j += 1
        pages.append((i, j - i, tot))
        i = j
    total = int(sizes.sum())
    first, count, nbytes = pages[0]
    ctx.grab_copy(first, count, nbytes)  # warm-up: module load, staging allocation
    ms = 0.0
    for _ in range(a.repeats):
        for first, count, nbytes in pages:
            ctx.grab_copy(first, count, nbytes)
            ms += ctx.timing()["grab_ms"]
    gathered = total * a.repeats
    rate = 2 * gathered / (ms / 1e3) if ms > 0 else 0.0
    name, limit = card()
    line = {"what": "k_grab, -S all on BASELINE configs[1]", "card": name, "power_limit": limit,
            "streams": a.streams, "packages": int(res["n_packages"]), "grabs": int(len(plan)), "bytes_gathered": total,
            "pages": len(pages), "repeats": a.repeats, "k_grab_ms_total": round(ms, 3),
            "k_grab_ms_per_pass": round(ms / a.repeats, 3), "hbm_GBps": round(rate / 1e9, 1),
            "share_of_3.35TBps": round(rate / PEAK_HBM, 3)}
    print(json.dumps(line))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
