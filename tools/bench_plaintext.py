#!/usr/bin/env python
"""Device-side rate of the plaintext side of Bfv: SIMD encode (Coeff and Eval), decode (Coeff and Eval) and
ciphertext + plaintext, through the _device entry points, timed with CUDA events after warm-up.  Prints one JSON line
per case with items/s and the achieved bandwidth on the compulsory bytes (DESIGN.md section 4) against the H100 SXM
data-sheet 3.35 TB/s, plus the card name and power limit read in the same run.

    python tools/bench_plaintext.py [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch

import hecuda

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]  # bench.py C2 (4 x 55 bits)
Q4096 = [134176769, 268369921, 268361729]                                            # 27/28/28 bits


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:  # reported, not guessed
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"


def timed(fn, reps):
    for _ in range(3):
        fn()
    s = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(reps):
        fn()
    e1.record(s)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / 1e3


def run(label, n, moduli, t, word_bytes, count, translate_batch, reps, name, limit, scalar=np.uint64):
    ctx = hecuda.Context(n, moduli, t, scalar=scalar)
    lib, s = hecuda.load_library(), torch.cuda.current_stream().cuda_stream
    L = ctx.L
    dev = torch.device("cuda", 0)
    values = torch.randint(0, t, (count, n), dtype=torch.int64, device=dev)
    coeff = torch.empty_like(values)
    ev = torch.empty((count, L, n), dtype=torch.int64, device=dev)
    back = torch.empty_like(values)
    ct = torch.randint(0, min(moduli[:L]), (translate_batch, 2, L, n), dtype=torch.int64, device=dev)
    pts = values[:translate_batch].contiguous()
    w = word_bytes
    cases = [
        # (name, call, items, compulsory bytes per item, composed-path rows moved per item)
        ("encode_coeff", lambda: lib.hecuda_bfv_encode_simd_device(ctx._h, values.data_ptr(), n, 0, coeff.data_ptr(), count, s),
         count, 2 * n * w, 4),
        (f"encode_eval_l{L}", lambda: lib.hecuda_bfv_encode_simd_device(ctx._h, values.data_ptr(), n, L, ev.data_ptr(), count, s),
         count, (1 + L) * n * w, 5 + 3 * L),
        ("decode_coeff", lambda: lib.hecuda_bfv_decode_simd_device(ctx._h, coeff.data_ptr(), 0, back.data_ptr(), count, s),
         count, 2 * n * w, 4),
        (f"decode_eval_l{L}", lambda: lib.hecuda_bfv_decode_simd_device(ctx._h, ev.data_ptr(), L, back.data_ptr(), count, s),
         count, 2 * n * w, 10),
        (f"translate_add_l{L}_in_place", lambda: lib.hecuda_bfv_plaintext_translate_device(
            ctx._h, ct.data_ptr(), 2, L, pts.data_ptr(), translate_batch, 0, ct.data_ptr(), translate_batch, s),
         translate_batch, (1 + 2 * L) * n * w, 1 + 2 * L),
    ]
    for case, fn, items, compulsory, rows in cases:
        sec = timed(lambda: hecuda._check(fn()), reps)
        print(json.dumps({
            "metric": f"plaintext {case}", "config": label, "items": items, "ms": round(sec * 1e3, 3),
            "items_per_s": round(items / sec), "compulsory_bytes_per_item": compulsory,
            "achieved_tb_s": round(items * compulsory / sec / 1e12, 3),
            "share_of_3.35_tb_s": round(items * compulsory / sec / HBM_BYTES_PER_S, 3),
            "rows_moved_per_item": rows, "gpu": name, "power_limit": limit}), flush=True)
    # correctness guard on what was timed: decode of the encoded values gives the values back
    hecuda._check(lib.hecuda_bfv_decode_simd_device(ctx._h, coeff.data_ptr(), 0, back.data_ptr(), count, s))
    torch.cuda.synchronize()
    assert torch.equal(back, values), label
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_plaintext.py needs a CUDA device")
    name, limit = card()
    # C2's context (bench.py): N = 8192, 4 x 55-bit coefficient moduli (L = 3), t = 557057
    run("C2 context: N=8192, L=3 x 55-bit, t=557057", 8192, Q8192, 557057, 8, 8192, 1024, args.reps, name, limit)
    # the reference's PIR default moduli, N = 4096, t = 65537, as Bfv<UInt64> and Bfv<UInt32> contexts.  The _device
    # entry points keep residues as 64-bit words for both (the uint32 buffers exist at the host boundary only).
    run("Bfv<UInt64> N=4096, 27/28/28-bit, t=65537", 4096, Q4096, 65537, 8, 8192, 4096, args.reps, name, limit)
    run("Bfv<UInt32> N=4096, 27/28/28-bit, t=65537 (64-bit device words)", 4096, Q4096, 65537, 8, 8192, 4096, args.reps,
        name, limit, scalar=np.uint32)


if __name__ == "__main__":
    main()
