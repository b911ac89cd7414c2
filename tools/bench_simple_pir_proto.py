"""SimplePIR requests and responses in the reference's protobuf messages on the device
(SimplePirShardedServer.computeResponsesProto, hecuda_simple_pir_compute_response_proto) against the host composition
it replaces: google.protobuf decode of every SimplePIRRequest, one hecuda_simple_pir_compute_response_shards call, and
google.protobuf encode of every SimplePIRResponse.

Shapes A and B of tools/bench_simple_pir_shards.py (5 shards, N = 2048, pt = 14, ct = 42, 64-bit words), with random
DB' values of the shards' computingParams shapes.  Every client sends ShardMap.chunksPerShard = 1 request (chunksPerEntry
rows) to every shard, so a call has 5 x clients messages; all clients send the same request bytes, which changes nothing
on the device.  One JSON line per shape and client count: clients/s for both paths (host clock, median of --reps after
a warm-up), the decode and encode kernel times (torch.profiler) and their bytes/s against 3.35 TB/s, the PCIe bytes per
client (messages and responses against words), the launches per call, and the card's name and power limit, read in the
same run.  The host composition is skipped ("not measured") past --host-limit message bytes per call."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tests")]

import hecuda  # noqa: E402
from hecuda import simple_pir as sp  # noqa: E402

SHAPES = {"A": (1 << 20, 52), "B": (4096, 52429)}  # rows per shard, chunk bytes
SHARDS = 5
HBM = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def classes():
    import test_simple_pir_proto as t
    return t.protobuf_classes()


def median_s(fn, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return statistics.median(times)


def kernel_ms(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "proto_" in e.name:
            key = "decode" if any(k in e.name for k in ("count", "decode", "check")) else \
                  "encode" if any(k in e.name for k in ("length", "write")) else "scan"
            out[key] = out.get(key, 0.0) + e.device_time / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="A,B")
    ap.add_argument("--clients", default="1,16,256")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-limit", type=float, default=6e8)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    name = card()
    cls = classes()
    rng = np.random.default_rng(0)
    enc = sp.SimplePirEncryptionParams(14, 42, 2048, 6.4)
    for shape in args.shapes.split(","):
        rows, chunk = SHAPES[shape]
        params = [sp.SimplePirParameters.computingParams(enc, rows, chunk, bytes(32)) for _ in range(SHARDS)]
        dbs = [sp.SimplePirDatabase.create(rng.integers(0, 1 << 14, size=(p.columnSize, p.databaseColumns), dtype=np.uint64),
                                           p) for p in params]
        server = sp.SimplePirShardedServer(dbs, [np.zeros((p.columnSize, 2048), np.uint64) for p in params], params)
        requests = [rng.integers(0, 1 << 42, size=(p.chunksPerEntry, p.databaseColumns), dtype=np.uint64) for p in params]
        per_client = [sp.SimplePirRequest.write(r, s) for s, r in enumerate(requests)]
        words_in = sum(r.size for r in requests) * 8
        words_out = sum(p.chunksPerEntry * p.columnSize for p in params) * 8
        for clients in [int(c) for c in args.clients.split(",")]:
            messages = per_client * clients
            server.computeResponsesProto(messages)  # warm-up
            t_proto = median_s(lambda: server.computeResponsesProto(messages), args.reps)
            before = hecuda.kernel_launch_count()
            replies = server.computeResponsesProto(messages)
            launches = hecuda.kernel_launch_count() - before
            kernels = kernel_ms(torch, lambda: server.computeResponsesProto(messages))
            msg_bytes = sum(len(m) for m in per_client)
            reply_bytes = sum(len(r) for r in replies[:SHARDS])
            host = None
            if msg_bytes * clients <= args.host_limit:
                def composition():
                    flat = np.empty((clients, words_in // 8), np.uint64)
                    for c in range(clients):
                        at = 0
                        for s in range(SHARDS):
                            m = cls["SimplePIRRequest"]()
                            m.ParseFromString(messages[c * SHARDS + s])
                            d = np.array(m.request.data, dtype=np.uint64)
                            flat[c, at:at + d.size] = d
                            at += d.size
                    out = server.computeResponses(flat, requests_per_shard=1)
                    encoded = []
                    for c in range(clients):
                        at = 0
                        for p in params:
                            n = p.chunksPerEntry * p.columnSize
                            r = cls["SimplePIRResponse"]()
                            r.response.row_count, r.response.col_count = p.chunksPerEntry, p.columnSize
                            r.response.data.extend(out[c, at:at + n].tolist())
                            encoded.append(r.SerializeToString())
                            at += n
                    return encoded
                assert composition() == replies, "the host composition's bytes differ"
                host = median_s(composition, args.reps)
            dec, encd = kernels.get("decode"), kernels.get("encode")
            print(json.dumps({
                "shape": shape, "clients": clients, "messages": len(messages),
                "proto_clients_per_s": round(clients / t_proto, 2),
                "host_clients_per_s": round(clients / host, 2) if host else "not measured",
                "decode_kernel_ms": round(dec, 3) if dec else None,
                "decode_GBps": round(msg_bytes * clients / (dec / 1e3) / 1e9, 1) if dec else None,
                "encode_kernel_ms": round(encd, 3) if encd else None,
                "encode_GBps": round(reply_bytes * clients / (encd / 1e3) / 1e9, 1) if encd else None,
                "scan_kernel_ms": round(kernels.get("scan", 0.0), 3), "hbm_TBps": HBM / 1e12,
                "pcie_in_bytes_per_client": {"messages": msg_bytes, "words": words_in},
                "pcie_out_bytes_per_client": {"messages": reply_bytes, "words": words_out},
                "launches_per_call": launches, "card": name}), flush=True)
        server.close()
        del dbs, server
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
