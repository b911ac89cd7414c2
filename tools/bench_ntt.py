#!/usr/bin/env python
"""NTT-only timing on one GPU (development tool): forward / inverse over the extended base [Q, Bsk] of config C2.
   python tools/bench_ntt.py [polys]"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "swift-homomorphic-encryption_b200"))
import torch, hecuda
from bench import workload_params
name = os.environ.get("WORKLOAD", "C2")
BASE = hecuda.BASE_Q_BSK if os.environ.get("NTT_BASE") == "bsk" else hecuda.BASE_Q_AUX
n, moduli, t, _ = workload_params(name)
polys = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
ctx = hecuda.Context(n, moduli, t); lib = hecuda.load_library(); L = ctx.L; R = 2 * L + 1
dev = torch.device("cuda", 0)
ext = torch.randint(0, 1 << 50, (polys, R, n), device=dev, dtype=torch.int64)
s = torch.cuda.current_stream()
out = {}
for label, fn in (("fwd", lib.hecuda_ntt_forward_device), ("inv", lib.hecuda_ntt_inverse_device)):
    for _ in range(3): fn(ctx._h, BASE, ext.data_ptr(), R, polys, s.cuda_stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record(s)
    reps = 10
    for _ in range(reps): fn(ctx._h, BASE, ext.data_ptr(), R, polys, s.cuda_stream)
    e1.record(s); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    out[label] = {"rows": polys * R, "ms": round(ms, 4), "Mrows_per_s": round(polys * R / ms / 1e3, 3), "GBps": round(polys * R * 2 * n * 8 / ms / 1e6, 1)}
print(json.dumps({"workload": name, "n": n, "polys": polys, **out}))
