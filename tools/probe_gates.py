#!/usr/bin/env python
"""Derive the decoder length gates (SURVEY 8(f1)) from the UNMODIFIED reference decoders (oracle/_ref) and write
rtl_433_b200/data/gates_25.12.json: for every protocol the largest T <= MAX_BITS such that every probed event whose
rows all hold fewer than T bits is rejected by decode_fn with one constant code c <= 0 and no output (exhaustive over
single rows, sampled over multi-row buffers: oracle/ref_harness.c:refh_probe_gate).  An r433b_gate {T, c} lets k_slice2
drop such events on the device and only count them (one-row and several-row events separately: many decoders test
num_rows first); the host adds the counts to decode_events / decode_fails[-code], so
the decoders' statistics stay what account_event() (src/pulse_slicer.c:26-66) would have produced.  Run in the build
container; tests/test_gates.py re-validates the committed table against the compiled reference with fresh inputs."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refh  # noqa: E402

MAX_BITS = 16
N_RANDOM = 3000


def main():
    L = refh.lib()
    L.refh_probe_gate.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.POINTER(C.c_int)]
    r = refh.Ref(store_bitbuffers=False)
    n = L.refh_num_protocols(r.h)
    for i in range(n):
        r.register(i + 1)
    devs = r.registered()
    gates = {}
    hist = {}
    for idx, d in enumerate(devs):
        code = (C.c_int * 2)()
        t = L.refh_probe_gate(r.h, idx, MAX_BITS, N_RANDOM, 1, code)
        gates[str(d["protocol_num"])] = [t, code[0], code[1]]
        hist[t] = hist.get(t, 0) + 1
    out = {"reference": "merbanan/rtl_433 25.12", "max_bits": MAX_BITS, "n_random": N_RANDOM,
           "doc": "protocol_num -> [T, code1, codeN]: events (>= 1 row) whose rows all hold < T bits make decode_fn return code1 (one row) / codeN (several rows)",
           "gates": gates}
    path = os.path.join(ROOT, "rtl_433_b200", "data", "gates_25.12.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, separators=(",", ":"))
    print(path, len(gates), "protocols; T histogram:", dict(sorted(hist.items())))
    codes = {}
    for t, c, cn in gates.values():
        codes[(c, cn)] = codes.get((c, cn), 0) + 1
    print("codes:", codes)


if __name__ == "__main__":
    main()
