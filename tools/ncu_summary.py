#!/usr/bin/env python
"""Summarise an .ncu-rep (read here, no GPU needed): headline metrics + hottest source lines."""
import collections
import csv
import io
import json
import subprocess
import os
import sys
import os as _os
KF = ["-k", "regex:" + _os.environ["NCU_KERNEL"]] if _os.environ.get("NCU_KERNEL") else []

rep, out_md = sys.argv[1], sys.argv[2]
traffic_json = sys.argv[3] if len(sys.argv) > 3 else None
raw = subprocess.run(["ncu", "-i", rep] + KF + [ "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rows[0], rows[1], rows[2]
m = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__waves_per_multiprocessor", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__average_warp_latency_per_inst_issued.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct"]
kernel = m.get("Kernel Name", ("?", ""))[0]
lines = [f"# ncu summary: `{kernel}`", "", f"source report: `{rep}` (`ncu --set full --clock-control none --import-source on`)", "",
         "| metric | value | unit |", "|---|---|---|"]
for k in want:
    if k in m:
        lines.append(f"| {k} | {m[k][0]} | {m[k][1]} |")


def num(k):
    v, u = m[k]
    v = float(v)
    mult = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1, "ms": 1e-3, "us": 1e-6, "ns": 1e-9, "s": 1}.get(u, 1)
    return v * mult


rd, wr, dur = num("dram__bytes_read.sum"), num("dram__bytes_write.sum"), num("gpu__time_duration.sum")
lines += ["", f"DRAM traffic per launch: {rd / 1e9:.3f} GB read + {wr / 1e9:.3f} GB written = {(rd + wr) / 1e9:.3f} GB in {dur * 1e3:.2f} ms "
          f"(under the profiler) = {(rd + wr) / dur / 1e9:.1f} GB/s"]
if traffic_json:
    short = "k_front" if "k_front" in kernel else "k_detect" if "k_detect" in kernel else "k_slice2" if "k_slice2" in kernel else kernel
    wl = os.environ.get("NCU_WORKLOAD", "ook_cu8_250k")
    try:
        allt = json.load(open(traffic_json))
    except Exception:
        allt = {}
    allt.setdefault(wl, {})[short] = {"dram_bytes_per_launch": int(rd + wr), "dram_bytes_read": int(rd), "dram_bytes_write": int(wr),
                                       "duration_ms_under_profiler": round(dur * 1e3, 3), "report": os.path.basename(rep)}
    json.dump(allt, open(traffic_json, "w"), indent=1, sort_keys=True)
src = subprocess.run(["ncu", "-i", rep] + KF + [ "--page", "source", "--print-source", "cuda,sass", "--csv"], capture_output=True, text=True).stdout
cur, hd, agg = None, None, collections.OrderedDict()
for r in csv.reader(io.StringIO(src)):
    if not r:
        continue
    if r[0] == "File Path":
        cur = r[1].split("/")[-1]
        continue
    if r[0] == "Function Name":
        continue
    if r[0] == "Line No":
        hd = r
        continue
    if hd and r[0] != "":
        d = dict(zip(hd[:10], r[:10]))
        try:
            k = (cur, int(d["Line No"]))
            a = agg.setdefault(k, [0.0, 0.0, d["Source"]])
            a[0] += float(d["# Samples"] or 0)
            a[1] += float(d["Instructions Executed"] or 0)
        except Exception:
            pass
ts = sum(v[0] for v in agg.values()) or 1
ti = sum(v[1] for v in agg.values()) or 1
lines += ["", "## hottest source lines (stall samples / executed warp instructions)", "", "| samples | instr | where | source |", "|---|---|---|---|"]
import os  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_src_cache = {}


def source_text(fn, ln):
    if fn not in _src_cache:
        path = os.path.join(ROOT, "rtl_433_b200", "csrc", fn)
        _src_cache[fn] = open(path).read().split("\n") if os.path.exists(path) else []
    t = _src_cache[fn]
    return t[ln - 1].strip()[:100].replace("|", "\\|") if 0 < ln <= len(t) else "-"


for (fn, ln), (sm, ins, text) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:25]:
    lines.append(f"| {100 * sm / ts:.1f}% | {100 * ins / ti:.1f}% | {fn}:{ln} | `{source_text(fn, ln)}` |")
if "k_detect" in kernel:
    fn = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_funcs.py"), rep, "k_detectILi2"], capture_output=True, text=True).stdout
    lines += ["", "## by device function (tools/ncu_funcs.py; the phases of the walk are separate functions)", "", fn.rstrip()]
kind = "slice" if "k_slice2" in kernel else None
if kind:
    reg = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_regions.py"), rep, kind], capture_output=True, text=True).stdout
    lines += ["", "## by code region (tools/ncu_regions.py; IQ samples of the 4096 x 2^20 workload)", "", reg.rstrip()]
open(out_md, "w").write("\n".join(lines) + "\n")
print("\n".join(lines[:40]))
