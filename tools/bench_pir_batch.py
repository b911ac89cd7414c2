#!/usr/bin/env python
"""MulPir with many clients per call (hecuda_mulpir_compute_response_clients) against the one-query-per-call path, at
the C4 shape of tools/bench_pir.py (2^20 entries x 64 B, N = 4096, q = 27/28/28 bits, t = 17, uint32 database rows).

    python tools/bench_pir_batch.py [--clients 1,2,4,8,16,32] [--entries N] [--reps R] [--out DIR]

For each K: K distinct seeded clients (own evaluation key, own query).  Reports
  - device-resident queries/s: the _device call on device buffers, timed with CUDA events after warm-up;
  - end-to-end queries/s: the host call (copies in and out included);
  - the current path: K host threads, one single-client hecuda_mulpir_compute_response each, in the same run;
  - the first-dimension scan alone (torch.profiler over one _device call): bytes/s on the compulsory bytes (the
    database once plus the clients' query ciphertexts once, plus the sums written), multiply-accumulates/s, and HBM
    database bytes per query.
and checks that every batched reply equals the single-client reply of the same client.  Prints one JSON line per K and
the card's name and power limit, read in the same run.  Query and key values are uniform residues: the server's
arithmetic does not depend on them being well-formed."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")):
    sys.path.insert(0, p)
import ctypes as C

import numpy as np
import torch

import hecuda
from hecuda import pir

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28_logt_5 (EncryptionParameters.swift:357-367)
SCAN_KERNELS = ("inner_product_plain_small_clients_kernel", "inner_product_plain_clients_kernel",  # a group's scans
                "inner_product_plain_small_kernel", "inner_product_plain_kernel")  # a lone client's scans


def uniform(rng, moduli, shape_prefix, n):
    out = np.empty(tuple(shape_prefix) + (len(moduli), n), dtype=np.uint64)
    for i, q in enumerate(moduli):
        out[..., i, :] = rng.integers(0, q, size=tuple(shape_prefix) + (n,), dtype=np.uint64)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", default="1,2,4,8,16,32")
    ap.add_argument("--entries", type=int, default=1 << 20)
    ap.add_argument("--entry-size", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pir_batch needs a CUDA device")
    n, t = 4096, 17
    ctx = hecuda.Context(n, PIR_MODULI, t)
    L = ctx.L
    rng = np.random.default_rng(3)
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(args.entries, args.entry_size, 2, 1, True, "hybridCompression",
                                                            False), ctx)
    chunk_count = -(-param.encodedEntrySize // pir.bytesPerPlaintext(ctx))
    count = chunk_count * int(np.prod(param.dimensions))
    db = pir.ProcessedDatabase(ctx, rng.integers(0, t, size=(count, n), dtype=np.uint64), None, evalFormat=False)
    server = pir.MulPirServer(param, ctx, [db])
    ptr, nbytes = C.c_void_p(), C.c_uint64()
    hecuda._check(hecuda.load_library().hecuda_pir_database_device_buffer(db._h, C.byref(ptr), C.byref(nbytes)))
    db_bytes = int(nbytes.value)
    elements = param.evaluationKeyConfig.galoisElements
    qct = -(-param.expandedQueryCount // n)
    ks = [int(k) for k in args.clients.split(",")]
    kmax = max(ks)
    keys, queries = [], []
    for c in range(kmax):
        crng = np.random.default_rng(1000 + c)
        key = hecuda.EvaluationKey(ctx, uniform(crng, PIR_MODULI, (L, 2), n))
        for e in elements:
            key.setGaloisKey(e, uniform(crng, PIR_MODULI, (L, 2), n))
        keys.append(key)
        queries.append(uniform(crng, PIR_MODULI[:L], (qct, 2), n))
    queries = np.stack(queries)
    dim0, rows = param.dimensions[0], chunk_count * (int(np.prod(param.dimensions)) // param.dimensions[0])
    lib = hecuda.load_library()
    handles = (C.c_void_p * 1)(db._h)
    dims = (C.c_int32 * len(param.dimensions))(*param.dimensions)
    info = dict(card=card(), dims=param.dimensions, chunk_count=chunk_count, database_bytes=db_bytes)
    print(json.dumps(info), flush=True)
    stream = torch.cuda.Stream()
    results = []
    for k in ks:
        key_handles = (C.c_void_p * k)(*[x._h for x in keys[:k]])
        with torch.cuda.stream(stream):
            d_q = torch.from_numpy(queries[:k].view(np.int64)).cuda()
            d_out = torch.empty((k, 1, chunk_count, 2, 1, n), dtype=torch.int64, device="cuda")
        stream.synchronize()

        def device_call():
            hecuda._check(lib.hecuda_mulpir_compute_response_clients_device(
                ctx._h, key_handles, k, handles, 1, dims, len(param.dimensions), chunk_count, d_q.data_ptr(), qct, 1,
                d_out.data_ptr(), stream.cuda_stream))

        for _ in range(2):
            device_call()
        stream.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        for _ in range(args.reps):
            device_call()
        end.record(stream)
        end.synchronize()
        device_ms = start.elapsed_time(end) / args.reps
        # the host call
        server.computeResponses(queries[:k], keys[:k])
        t0 = time.perf_counter()
        for _ in range(args.reps):
            batched = server.computeResponses(queries[:k], keys[:k])
        host_ms = (time.perf_counter() - t0) * 1e3 / args.reps
        # the current path: k threads, one single-client call each
        singles = [None] * k

        def worker(c, reps):
            for _ in range(reps):
                singles[c] = server.computeResponse(queries[c], keys[c])

        for reps in (2, args.reps):
            pool = [threading.Thread(target=worker, args=(c, reps)) for c in range(k)]
            t0 = time.perf_counter()
            for th in pool:
                th.start()
            for th in pool:
                th.join()
            threads_ms = (time.perf_counter() - t0) * 1e3 / reps
        same = all(np.array_equal(batched[c], singles[c]) for c in range(k))
        same_device = np.array_equal(d_out.cpu().numpy().view(np.uint64), batched)
        # the scan alone
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            device_call()
            stream.synchronize()
        scan_us = [e.device_time_total for e in prof.key_averages() if any(s in e.key for s in SCAN_KERNELS)]
        scan_ms = sum(scan_us) / 1e3 if scan_us else float("nan")
        groups = -(-k // 16)
        query_bytes = k * dim0 * 2 * L * n * 8
        out_bytes = k * rows * 2 * L * n * 8
        macs = k * rows * dim0 * 2 * L * n
        res = dict(clients=k, device_ms=round(device_ms, 3), device_qps=round(k / device_ms * 1e3, 1),
                   host_ms=round(host_ms, 3), host_qps=round(k / host_ms * 1e3, 1),
                   threads_ms=round(threads_ms, 3), threads_qps=round(k / threads_ms * 1e3, 1),
                   scan_ms=round(scan_ms, 4),
                   scan_compulsory_GBps=round((groups * db_bytes + query_bytes + out_bytes) / scan_ms / 1e6, 1),
                   scan_GMACps=round(macs / scan_ms / 1e6, 1),
                   hbm_db_bytes_per_query=int(groups * db_bytes / k),
                   batched_equals_single=bool(same), device_equals_host=bool(same_device))
        results.append(res)
        print(json.dumps(res), flush=True)
        assert same and same_device, "batched replies differ from the single-client replies"
    print(json.dumps(dict(card=card(), results=results)), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_pir_batch.json"), "w") as f:
            json.dump(dict(info, results=results), f, indent=1)


if __name__ == "__main__":
    main()
