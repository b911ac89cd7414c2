"""SimplePIR's device client (hecuda.simple_pir.DefaultQueryGenerator / SimplePirClient) at the two shapes of
tools/bench_simple_pir.py, N = 2048, errorStdDev 6.4, pt = 14, ct = 42:

  A  2^20 entries x 256 B     M = 147,    K = 1 048 576
  B  4096 entries x 256 KiB   M = 24 967, K = 24 576, chunksPerEntry 6

One JSON line per shape: precompute queries/s at 1, 16 and 256 queries through the host call and the device call
(CUDA events), per-kernel device time of one 16-query device call (torch.profiler, kernels grouped as the DRBG chains,
the ternary kernel, the NTTs, the pointwise products, the finish kernel and the results product), decrypts/s of the
device call at 256, and the results product's int8 op/s (2 x 2 masks x ceil((ct + 1) / 8) planes x M x N x secret rows)
with its share of the 1,979 TOPS dense data-sheet figure and of the hint-plane read at 3.35 TB/s.  A further line gives
SimplePirShardedServer.validate's wall time on a 5-shard database and a parity check of a reduced shape (N 2048,
K 4096) against tests/simple_pir_client_ref.py (the Python AES is too slow for shape A).  The card's name and power
limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tests")]

import hecuda  # noqa: E402
from hecuda import simple_pir as sp  # noqa: E402

SHAPES = {"A": (1 << 20, 256), "B": (4096, 256 * 1024)}
GROUPS = [("drbg", "drbg_chain"), ("ternary", "ternary_kernel"), ("ntt", "ntt"), ("pointwise", "pointwise_kernel"),
          ("finish", "finish_kernel"), ("results", "results_kernel")]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def seeds(count):
    return np.frombuffer(os.urandom(32 * count), dtype=np.uint8).copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="A,B")
    ap.add_argument("--batches", default="1,16,256")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    hecuda.set_device(0)
    name = card()
    enc = sp.SimplePirEncryptionParams(14, 42, 2048, 6.4)
    for label in args.shapes.split(","):
        count, size = SHAPES[label]
        rng = np.random.default_rng(1)
        entries = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
        res = sp.SimplePirServer.process(entries, enc, seed=bytes(32))
        prm = res.params
        gen = sp.DefaultQueryGenerator(prm, res.hint)
        client = sp.SimplePirClient(gen)
        m, k, cpe, n = prm.columnSize, prm.databaseColumns, prm.chunksPerEntry, prm.latticeDimension
        planes = (42 + 1 + 7) // 8
        row = {"shape": label, "card": name, "M": m, "K": k, "chunksPerEntry": cpe}
        stream = torch.cuda.current_stream().cuda_stream
        for b in [int(x) for x in args.batches.split(",")]:
            gen.precompute(b)
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                gen.precompute(b)
                times.append(time.perf_counter() - t0)
            d_ss, d_es = torch.from_numpy(seeds(b)).cuda(), torch.from_numpy(seeds(b)).cuda()
            d_q = torch.empty((b, cpe, k), dtype=torch.int64, device="cuda")
            d_r = torch.empty((b, cpe, m), dtype=torch.int64, device="cuda")

            def call():
                client.precomputeDevice(d_ss.data_ptr(), d_es.data_ptr(), None, b, d_q.data_ptr(), d_r.data_ptr(), stream)

            call()
            dev = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                torch.cuda.synchronize()
                dev.append(e0.elapsed_time(e1) * 1e-3)
            row[f"host_queries_per_s_{b}"] = round(b / statistics.median(times), 2)
            row[f"device_queries_per_s_{b}"] = round(b / statistics.median(dev), 2)
            row[f"device_ms_{b}"] = round(statistics.median(dev) * 1e3, 3)
            if b == 16:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call()
                    torch.cuda.synchronize()
                per = defaultdict(float)
                for ev in prof.events():
                    if ev.device_type.name != "CUDA":
                        continue
                    for group, key in GROUPS:
                        if key in ev.name:
                            per[group] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                            break
                row["kernel_us_16"] = {g: round(per[g], 1) for g, _ in GROUPS}
                results_s = per["results"] * 1e-6
                ops = 2 * 2 * planes * m * n * b * cpe
                if results_s > 0:
                    row["results_int8_ops_per_s_16"] = ops / results_s
                    row["results_share_of_1979_tops_16"] = round(ops / results_s / 1.979e15, 4)
                    row["results_share_of_hint_read_16"] = round(planes * m * n / 3.35e12 / results_s, 4)
            if b == max(int(x) for x in args.batches.split(",")):
                idx = torch.zeros(b, dtype=torch.int64, device="cuda")
                d_out = torch.empty((b, prm.entrySizeInBytes), dtype=torch.uint8, device="cuda")
                client.decryptDevice(d_r.data_ptr(), d_r.data_ptr(), idx.data_ptr(), b, d_out.data_ptr(), stream)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    client.decryptDevice(d_r.data_ptr(), d_r.data_ptr(), idx.data_ptr(), b, d_out.data_ptr(), stream)
                e1.record()
                torch.cuda.synchronize()
                row[f"decrypts_per_s_{b}"] = round(b * args.reps / (e0.elapsed_time(e1) * 1e-3), 1)
                del idx, d_out
            del d_ss, d_es, d_q, d_r
        print(json.dumps(row), flush=True)
        gen.close()
        res.database.close()

    import simple_pir_client_ref as ref
    rng = np.random.default_rng(2)
    entries = rng.integers(0, 256, size=(2000, 1024), dtype=np.uint8)
    server = sp.SimplePirShardedServer.process(entries, enc, 5, rng=rng)
    index = 17
    server.validate((index, entries[index].tobytes()))
    t0 = time.perf_counter()
    times, _ = server.validate((index, entries[index].tobytes()), trials=3)
    wall = (time.perf_counter() - t0) / 3
    prm = sp.SimplePirParameters(enc, 64, 1, 1, 4096, bytes(range(32)))
    hint = rng.integers(0, 1 << 40, size=(prm.columnSize, 2048), dtype=np.uint64)
    gen = sp.DefaultQueryGenerator(prm, hint)
    ss, es = [os.urandom(32)], [os.urandom(32)]
    q, r = gen.precompute(1, [5], ss, es)
    d = dict(N=2048, pt=14, ct=42, entries_per_column=1, chunks_per_entry=1, database_columns=4096)
    eq, er, _ = ref.precompute(d, hint, prm.seed, ss[0], es[0], 5, 64, 6.4)
    parity = "ok" if np.array_equal(q[0], eq) and np.array_equal(r[0], er) else "MISMATCH"
    print(json.dumps({"card": name, "validate_5_shards_s": round(wall, 4), "validate_round_trip_s": [round(t, 4) for t in times],
                      "parity_reduced_shape": parity}), flush=True)


if __name__ == "__main__":
    main()
