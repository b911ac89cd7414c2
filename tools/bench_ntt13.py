#!/usr/bin/env python
"""The two N = 2^13 NTT kernels of the C2 multiply, timed on one GPU (development tool).

    python tools/bench_ntt13.py [--workload C2] [--pairs 1024] [--reps 10] [--tree DIR]

- CUDA events around the row NTT kernel (ntt_rows_kernel<13, ...>) at the multiply's launch shapes: the inverse over
  3 R rows per pair of one pipeline stage, and the forward over 4 R rows per pair (the operand rows the fused kernel
  transforms), both over [Q, aux];
- torch.profiler over whole multiply steps (`pairs` ciphertext pairs): per-kernel device time per step, which names the
  fused forward NTT + tensor kernel (ntt_forward_tensor_kernel<13, ...>) and the inverse;
- the L2-side bytes a row reads: the row, plus the LB == 0 pass's transposed twiddles (120 KB) when they come from global
  memory, or the resident twiddle image (96 KB) amortised over the rows a CTA runs per modulus when they are kept in
  shared memory.

--tree DIR imports hecuda (and its libhecuda.so) from another checkout, so two builds can be timed in one session.
Prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="C2")
ap.add_argument("--pairs", type=int, default=1024)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--tree", default=ROOT)
args = ap.parse_args()
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.abspath(args.tree), "swift-homomorphic-encryption_b200"))

import torch  # noqa: E402
import hecuda  # noqa: E402
from bench import workload_params  # noqa: E402

n, moduli, t, _ = workload_params(args.workload)
assert n == 8192, "the resident twiddle image is the N = 2^13 kernels'"
ctx = hecuda.Context(n, moduli, t)
lib = hecuda.load_library()
L = ctx.L
R = 2 * L + 1
dev = torch.device("cuda", 0)
s = torch.cuda.current_stream()
sms = torch.cuda.get_device_properties(0).multi_processor_count
# pipeline stage of the multiply (capi.cu): ~2 GB of scratch at 7 R N words a pair
stage = min(args.pairs, max(1, (2048 * 1024 * 1024) // (7 * R * n * 8)))


def check(rc):
    assert rc == 0, lib.hecuda_last_error()


def timed(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(s)
    for _ in range(reps):
        fn()
    e1.record(s)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


out = {"workload": args.workload, "tree": os.path.abspath(args.tree), "gpu": torch.cuda.get_device_name(0),
       "pairs": args.pairs, "pipeline_stage_pairs": stage}
rows = {}
for label, polys, fn in (("inverse", 3 * stage, lib.hecuda_ntt_inverse_device), ("forward", 4 * stage, lib.hecuda_ntt_forward_device)):
    data = torch.randint(0, 1 << 50, (polys, R, n), device=dev, dtype=torch.int64)
    ms = timed(lambda: check(fn(ctx._h, hecuda.BASE_Q_AUX, data.data_ptr(), R, polys, s.cuda_stream)), args.reps)
    rows[label] = polys * R
    out[f"rows_{label}"] = {"rows": polys * R, "ms": round(ms, 4), "ns_per_row": round(ms * 1e6 / (polys * R), 1)}
    del data

# L2-side bytes per row: a CTA runs about rows / (grid x moduli) consecutive rows of one modulus
row_bytes, tw_t_bytes, image_bytes = 8 * n, 15 * (n // 16) * 16, 12 * (n // 16) * 16
rows_per_reload = rows["inverse"] / (sms * R)
out["l2_bytes_per_row"] = {
    "global_transposed_table": row_bytes + tw_t_bytes,
    "resident_image": round(row_bytes + image_bytes / rows_per_reload),
    "rows_per_image_reload": round(rows_per_reload, 1),
}

# whole multiply steps under the profiler: device time per kernel per step
qs = torch.tensor(moduli[:L], dtype=torch.int64, device=dev).view(1, 1, L, 1)
lhs = torch.randint(0, 1 << 62, (args.pairs, 2, L, n), device=dev, dtype=torch.int64) % qs
rhs = torch.randint(0, 1 << 62, (args.pairs, 2, L, n), device=dev, dtype=torch.int64) % qs
prod = torch.empty((args.pairs, 3, L, n), dtype=torch.int64, device=dev)


def step():
    check(lib.hecuda_bfv_multiply_device(ctx._h, lhs.data_ptr(), rhs.data_ptr(), prod.data_ptr(), args.pairs, s.cuda_stream))


out["multiply_step_ms"] = round(timed(step, args.reps), 4)
from torch.profiler import ProfilerActivity, profile  # noqa: E402

torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.reps):
        step()
    torch.cuda.synchronize()
kernels = {}
for ev in prof.key_averages():
    if ev.device_type.name == "CUDA" and ev.count:
        name = ev.key.split("(")[0].replace("void ", "")
        total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total")
        kernels[name] = round(kernels.get(name, 0.0) + total / 1e3 / args.reps, 4)
out["kernel_ms_per_step"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]))
print(json.dumps(out))
