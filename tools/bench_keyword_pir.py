"""Keyword-PIR processing and response times (KeywordPirServer.processOnDevice, KeywordPirServer.computeResponse[s]).

Shapes (synthetic, seeded; 16-byte keywords, SplitMix64 evictions, defaultKeywordPir cuckoo tables, 2 dimensions):
  100 000 x 2 B and 1 000 x 60 000 B at n_4096_logq_27_28_28_logt_4 (t = 11) and _logt_5 (t = 17)
  (EncryptionParameters.swift:346-367), and 2^20 x 64 B at the C4 context (N = 4096, t = 17, 27/28/28-bit moduli).

Per shape one JSON line:
  - process_ms: wall time of processOnDevice through Python (keyword/value concatenation, table, databases), ending in a
    device synchronise; `reps` runs after one warm-up;
  - kernels_ms: the device kernels of one processOnDevice from torch.profiler, in a separate pass;
  - python_oracle_ms: the CPU oracle (oracle/keyword_oracle.py) building and serializing the same table -- a Python
    restatement, not the reference -- for shapes up to --oracle-max-rows rows;
  - at 100 000 x 2 B: the response time of one keyword query and of a group of 16 clients.
The first line names the card and its power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")]

import hecuda  # noqa: E402
from hecuda import keyword_pir as kw  # noqa: E402

PIR_MODULI = [134176769, 268369921, 268361729]
LOGT = {11: "n_4096_logq_27_28_28_logt_4", 17: "n_4096_logq_27_28_28_logt_5"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "error": str(e)}


def rows_for(count, size, seed):
    rng = np.random.default_rng(seed)
    keywords = rng.integers(0, 256, size=(count, 16), dtype=np.uint8)
    values = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
    return [(keywords[i].tobytes(), values[i].tobytes()) for i in range(count)]


def sync():
    import torch
    torch.cuda.synchronize()


def bench_shape(name, ctx, rows, value_size, reps, oracle_max_rows):
    bpp = ctx.degree * (ctx.plaintextModulus.bit_length() - 1) // 8
    single = kw.serializedSize(value_size)
    bucket = -(-single // bpp) * bpp if single >= bpp // 2 else bpp // 2   # defaultMaxSerializedBucketSize
    config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(bucket), False, "hybridCompression")
    processed = kw.KeywordPirServer.processOnDevice(rows, config, ctx, kw.Rng.splitMix64(1))
    processed.close()
    times = []
    for _ in range(reps):
        sync()
        t0 = time.perf_counter()
        processed = kw.KeywordPirServer.processOnDevice(rows, config, ctx, kw.Rng.splitMix64(1))
        sync()
        times.append((time.perf_counter() - t0) * 1e3)
        info = processed.table.summarize()
        param = processed.pirParameter
        processed.close()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kw.KeywordPirServer.processOnDevice(rows, config, ctx, kw.Rng.splitMix64(1)).close()
        sync()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
            kernels[ev.key.split("(")[0][-40:]] = round(t / 1e3, 3)
    out = {"shape": name, "rows": len(rows), "value_bytes": value_size, "N": ctx.degree, "t": ctx.plaintextModulus,
           "maxSerializedBucketSize": bucket, "buckets": info.bucketCount, "loadFactor": float(info.loadFactor),
           "entry_size": param.entrySizeInBytes, "dims": param.dimensions,
           "process_ms": [round(t, 1) for t in times], "kernels_ms": kernels, "kernels_total_ms": round(sum(kernels.values()), 3)}
    if len(rows) <= oracle_max_rows:
        from oracle import keyword_oracle as K
        t0 = time.perf_counter()
        K.CuckooTable(K.CuckooTableConfig(2, 100, bucket), rows, K.SplitMix64(1)).serialize_buckets()
        out["python_oracle_table_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    else:
        out["python_oracle_table_ms"] = "not run (above --oracle-max-rows)"
    return out, config


def bench_response(ctx, rows, config, reps):
    from oracle import keyword_oracle as K
    from oracle import oracle as orc
    from oracle import pir_oracle as opir
    o = orc.Context(ctx.degree, PIR_MODULI, ctx.plaintextModulus)
    processed = kw.KeywordPirServer.processOnDevice(rows, config, ctx, kw.Rng.splitMix64(1))
    server = kw.KeywordPirServer(ctx, processed)
    param = processed.pirParameter
    oparam = opir.generate_parameter(opir.IndexPirConfig(param.entryCount, param.entrySizeInBytes, 2, 2, False,
                                                         "hybridCompression", False), o.n, o.t)
    keys, queries = [], []
    for c in range(16):
        sk, relin = o.keygen(50 + c)
        key = hecuda.EvaluationKey(ctx, relin)
        for i, e in enumerate(param.evaluationKeyConfig.galoisElements):
            key.setGaloisKey(e, o.galois_keygen(500 + 31 * c + i, sk, e))
        keys.append(key)
        queries.append(np.stack(K.generate_query(o, oparam, rows[c][0], 2, sk, 900 + c)))
    server.computeResponse(queries[0], keys[0])
    server.computeResponses(np.stack(queries), keys)
    one, group = [], []
    for _ in range(reps):
        sync()
        t0 = time.perf_counter()
        server.computeResponse(queries[0], keys[0])
        sync()
        one.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        server.computeResponses(np.stack(queries), keys)
        sync()
        group.append((time.perf_counter() - t0) * 1e3)
    for k in keys:
        k.close()
    processed.close()
    return {"response_one_query_ms": [round(t, 2) for t in one], "response_16_clients_ms": [round(t, 2) for t in group],
            "reference_published": "keyword-PIR server runtime ~51 ms for 100 000 x 2 B rows (BASELINE.md section 1, "
                                   "the reference's own published figure on its own hardware)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-max-rows", type=int, default=100000)
    ap.add_argument("--skip-c4", action="store_true")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    for t in (11, 17):
        ctx = hecuda.Context(4096, PIR_MODULI, t)
        for count, size in ((100000, 2), (1000, 60000)):
            out, config = bench_shape(f"{count}x{size}B {LOGT[t]}", ctx,
                                      rows_for(count, size, count + t), size, args.reps, args.oracle_max_rows)
            if count == 100000:
                out.update(bench_response(ctx, rows_for(count, size, count + t), config, args.reps))
            print(json.dumps(out), flush=True)
        ctx.close()
    if not args.skip_c4:
        ctx = hecuda.Context(4096, PIR_MODULI, 17)
        out, _ = bench_shape("C4 2^20x64B", ctx, rows_for(1 << 20, 64, 4), 64, args.reps, args.oracle_max_rows)
        print(json.dumps(out), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
