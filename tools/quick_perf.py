#!/usr/bin/env python
"""Quick device-resident throughput probe (not the contract bench): N replicas of a few distinct
synthetic streams, inputs already in HBM, prints the library's own CUDA-event timings."""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtl_433_b200 import lib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=1024)
ap.add_argument("--distinct", type=int, default=32)
ap.add_argument("--log2n", type=int, default=20)
ap.add_argument("--fsk", action="store_true")
ap.add_argument("--devices", default="all")
ap.add_argument("--iters", type=int, default=3)
ap.add_argument("--pipeline", type=int, default=0)
ap.add_argument("--gates", action="store_true", help="decoder length gates on (r433b_set_gates)")
ap.add_argument("--bursts", type=int, default=0, help="bursts per OOK stream (0 = synth default)")
a = ap.parse_args()

n = 1 << a.log2n
t = time.time()
cache = f"/tmp/qp_{'fsk' if a.fsk else 'ook'}_{a.distinct}_{a.log2n}_{a.bursts}.npy"
if a.fsk:
    fmt, rate, freq = lib.FMT_CS16, 1024000, 868000000
else:
    fmt, rate, freq = lib.FMT_CU8, 250000, 433920000
if os.path.exists(cache):
    host = np.load(cache)
else:
    if a.fsk:
        base = [synth.fsk_stream(s, n_samples=n).view(np.uint8) for s in range(a.distinct)]
    else:
        kw = {"n_bursts": a.bursts} if a.bursts else {}
        base = [synth.ook_stream(s, n_samples=n, **kw) for s in range(a.distinct)]
    host = np.concatenate(base)
    np.save(cache, host)
print("generated", a.distinct, "streams in %.1fs" % (time.time() - t))
per = host.nbytes // a.distinct
dev_small = torch.from_numpy(host).cuda()
reps = (a.streams + a.distinct - 1) // a.distinct
dev = dev_small.repeat(reps)[: a.streams * per].contiguous()
offsets = (np.arange(a.streams + 1, dtype=np.uint64) * per)
devs = lib.default_device_table()
if a.devices != "all":
    devs = devs[: int(a.devices)]
ctx = lib.Context(0)
ctx.set_devices(devs)
if a.gates:
    ctx.set_gates(lib.default_gates(devs))
ctx.set_pipeline(a.pipeline)
import time as _t
torch.cuda.synchronize()
for it in range(a.iters):
    torch.cuda.synchronize(); _t0 = _t.perf_counter()
    ctx.process(dev.data_ptr(), offsets, fmt, rate, freq, data_on_device=True)
    torch.cuda.synchronize(); _wall = (_t.perf_counter() - _t0) * 1e3
    tm = ctx.timing()
    c = ctx.counts()
    ms = tm["detect_ms"] + tm["slice_ms"]
    print(f"iter {it}: front {tm['front_ms']:.2f} redone {tm['front_redone']} repaired {tm['front_repairs']} idle skipped {tm['idle_skipped']} rewalks {tm['idle_rewalks']} wall {_wall:.2f} ms ({c['samples'] / _wall / 1e3:.0f} MS/s) detect {tm['detect_ms']:.2f} ms  slice {tm['slice_ms']:.2f} ms  launches {tm['detect_launches']}+{tm['slice_launches']}  "
          f"packages {c['packages']} events {c['events']} event_bytes {c['event_bytes']}  "
          f"-> {c['samples'] / ms / 1e3:.1f} MS/s  detect-only {c['samples'] / tm['detect_ms'] / 1e3:.1f} MS/s "
          f"({c['samples'] * fmt / tm['detect_ms'] / 1e6:.1f} GB/s)")
t = time.time()
ctx.fetch()
print("fetch %.1f ms (d2h %.1f ms)" % ((time.time() - t) * 1e3, ctx.timing()["d2h_ms"]))
