#!/usr/bin/env python
"""Processing the server's databases: the host packing + upload against the device packing, at two shapes.

    python tools/bench_process_db.py [--reps R]

  C4: MulPirServer.process of 2^20 entries x 64 B, N = 4096, t = 17, 27/28/28-bit moduli, dimensions from
      generateParameter (two, uneven, hybridCompression).
      host   = plaintextRows (Python) + hecuda_pir_database_create(coefficients) + the synchronise
      device = hecuda_pir_database_create_from_entries (MulPirServer.processOnDevice) + the synchronise
  C5: PlaintextMatrix(signedValues:) of a 100 000 x 512 matrix in .diagonal packing, N = 8192, t = 65537, C5's moduli.
      host   = centeredToRemainder + diagonalPlaintexts (numpy) + hecuda_pnns_matrix_create(coefficients) + synchronise
      device = hecuda_pnns_matrix_create_from_values (PlaintextMatrix.fromSignedValues) + the synchronise

Synthetic, seeded data.  Per shape, one JSON line: wall times (one host run, `reps` device runs after one warm-up; at C4
also the Python argument building and the bare C call, each timed separately), the
bytes each path sends across PCIe, the device path's kernel times from torch.profiler, whether the two resident
buffers are identical, and the card and its power limit (read in the same run).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch

import hecuda
from hecuda import pir, pnns

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28_logt_5 (EncryptionParameters.swift:357-367)
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]


def card():
    """Name and power limit of the GPU, read-only."""
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in line.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as exc:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(exc)}


def device_words(ptr, nbytes):
    class Buffer:
        __cuda_array_interface__ = {"shape": (nbytes // 8,), "typestr": "<i8", "data": (ptr, False), "version": 2}

    return torch.as_tensor(Buffer(), device="cuda")


def kernel_times(fn):
    """fn() under torch.profiler: total device time per kernel name (ms), and fn's result."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    times = {}
    for evt in prof.key_averages():
        us = getattr(evt, "device_time_total", 0) or getattr(evt, "cuda_time_total", 0)
        if us and not evt.key.startswith("Memcpy") and not evt.key.startswith("Memset"):
            name = evt.key.replace("(anonymous namespace)::", "").split("(")[0][:80]
            times[name] = round(times.get(name, 0) + us / 1e3, 3)
    return times, result


def timed(fn, reps):
    fn().close()  # warm-up
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        obj = fn()
        torch.cuda.synchronize()
        out.append(round((time.perf_counter() - t0) * 1e3, 2))
        obj.close()
    return out


def bench_pir(reps):
    n, t, entries, size = 4096, 17, 1 << 20, 64
    ctx = hecuda.Context(n, PIR_MODULI, t)
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(entries, size, 2, 1, True, "hybridCompression"), ctx)
    raw = np.random.default_rng(4).integers(0, 256, size=(entries, size), dtype=np.uint8)
    database = [bytes(row) for row in raw]
    t0 = time.perf_counter()
    rows, present = pir.MulPirServer.plaintextRows(database, ctx, param)
    pack_s = time.perf_counter() - t0
    host = pir.ProcessedDatabase(ctx, rows, present)
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    host_pcie = rows.nbytes + present.nbytes
    del rows, present
    device_ms = timed(lambda: pir.MulPirServer.processOnDevice(database, ctx, param), reps)
    # the wrapper's two parts, each timed on its own: joining the Python bytes objects and building the offsets, and
    # the C call (upload, packing, Eval conversion, narrowing) with those arguments prepared beforehand
    arguments_ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        data, offsets, dims = pir._entry_arguments(database, param)
        arguments_ms.append(round((time.perf_counter() - t0) * 1e3, 2))

    def c_call():
        h = C.c_void_p()
        hecuda._check(hecuda.load_library().hecuda_pir_database_create_from_entries(
            ctx._h, hecuda._ptr(data), hecuda._ptr(offsets), entries, size, 0, dims, 2, C.byref(h)))
        return pir.ProcessedDatabase._adopt(ctx, h, host.count)

    c_call_ms = timed(c_call, reps)
    kernels, device = kernel_times(lambda: pir.MulPirServer.processOnDevice(database, ctx, param))
    same = bool(torch.equal(device_words(*device.deviceBuffer()), device_words(*host.deviceBuffer())))
    out = {"shape": "C4", "config": f"MulPir {entries} x {size} B, N={n}, t={t}, q=27/28/28 bit, dims={param.dimensions}",
           "plaintexts": host.count, "host_pack_s": round(pack_s, 2), "host_total_s": round(host_s, 2),
           "device_ms": device_ms, "python_arguments_ms": arguments_ms, "c_call_ms": c_call_ms, "host_pcie_bytes": int(host_pcie),
           "device_pcie_bytes": entries * size + (entries + 1) * 8,
           "device_kernels_ms": kernels, "resident_identical": same}
    host.close(), device.close()
    ctx.close()
    return out


def bench_pnns(reps):
    n, t, rows, cols = 8192, 65537, 100000, 512
    ctx = hecuda.Context(n, Q8192, t)
    dims = pnns.MatrixDimensions(rows, cols)
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(cols)
    values = np.random.default_rng(5).integers(-(t // 2), (t - 1) // 2 + 1, size=(rows, cols), dtype=np.int64)
    t0 = time.perf_counter()
    plain = pnns.PlaintextMatrix.diagonalPlaintexts(ctx, dims, bsgs, pnns.centeredToRemainder(values, t).reshape(-1))
    pack_s = time.perf_counter() - t0
    host = pnns.PlaintextMatrix(ctx, dims, None, bsgs, plaintexts=plain)
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    host_pcie = plain.nbytes
    del plain
    device_ms = timed(lambda: pnns.PlaintextMatrix.fromSignedValues(ctx, dims, values, bsgs), reps)
    kernels, device = kernel_times(lambda: pnns.PlaintextMatrix.fromSignedValues(ctx, dims, values, bsgs))
    same = bool(torch.equal(device_words(*device.deviceBuffer()), device_words(*host.deviceBuffer())))
    out = {"shape": "C5", "config": f"PNNS {rows} x {cols} signed values, N={n}, t={t}, 4 x 55-bit moduli, "
                                    f"babyStep={bsgs.babyStep}, giantStep={bsgs.giantStep}",
           "host_pack_s": round(pack_s, 2), "host_total_s": round(host_s, 2), "device_ms": device_ms,
           "host_pcie_bytes": int(host_pcie), "device_pcie_bytes": int(values.nbytes), "device_kernels_ms": kernels,
           "resident_identical": same}
    host.close(), device.close()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    hecuda.set_device(0)
    torch.cuda.set_device(0)
    info = card()
    results = [bench_pir(args.reps), bench_pnns(args.reps)]
    for r in results:
        r.update(info)
        print(json.dumps(r))
    if not all(r["resident_identical"] for r in results):
        raise SystemExit("device-processed resident buffers differ from the host-processed ones")


if __name__ == "__main__":
    main()
