"""Sharded SimplePIR on the device (hecuda.simple_pir.SimplePirShardedServer), as the SimplePIRProcessDatabase tool
deploys it: shardCount = 5 (the tool's default), N = 2048, errorStdDev 6.4, pt = 14, ct = 42.

  A  2^20 entries x 256 B,    chunk 52 B      (5 chunks an entry, 2^20 rows a shard)
  B  4096 entries x 256 KiB,  chunk 52 429 B  (5 chunks an entry, 4096 rows a shard)

One JSON line per shape and client count.  Every client sends ShardMap.chunksPerShard = 1 request to every shard.
grouped_*: one hecuda_simple_pir_compute_response_shards call for all clients and shards; serial_*: 5 calls of
hecuda_simple_pir_compute_response, one per shard, with the same requests.  *_host_ms is the host-pointer call
(upload, compute, download; a host clock around calls that synchronise), *_device_ms the device-pointer call (CUDA
events).  Medians of --reps runs after a warm-up at each shape.  The host calls are skipped (null) when a batch's
requests pass 2 GiB.  Parity: the grouped responses equal the serial ones for the first and last client, and
the first 4 DB' rows of every shard's response to client 0 equal the oracle's.

A "process" line per shape compares process_shards (values up once, shards gathered on the device) with the host
shardDatabase plus 5 SimplePirServer.process calls (each shard's byte matrix uploaded), with the bytes each path
sends over PCIe and the kernel launches of one call.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")]

import hecuda  # noqa: E402
from hecuda import simple_pir as sp  # noqa: E402
from oracle import simple_pir_oracle as osp  # noqa: E402

SHAPES = {"A": (1 << 20, 256, 52), "B": (4096, 256 * 1024, 52429)}
SHARDS = 5
HOST_LIMIT = 2 << 30


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def median_ms(fn, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(times), 3)


def median_event_ms(torch, fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return round(statistics.median(times), 3)


def launches(fn):
    before = hecuda.kernel_launch_count()
    fn()
    return hecuda.kernel_launch_count() - before


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="A,B")
    ap.add_argument("--clients", default="1,16,256")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    hecuda.set_device(0)
    name = card()
    enc = sp.SimplePirEncryptionParams(14, 42, 2048, 6.4)
    for label in args.shapes.split(","):
        count, size, chunk = SHAPES[label]
        rng = np.random.default_rng(1)
        entries = rng.integers(0, 256, size=(count, size), dtype=np.uint8)

        def device_process():
            return sp.SimplePirShardedServer.process(entries, enc, SHARDS, chunk, seed=bytes(32),
                                                     rng=np.random.default_rng(2))

        def host_process():
            _, shards = sp.DatabaseMap.shardDatabase(entries, SHARDS, chunk, rng=np.random.default_rng(2))
            return [sp.SimplePirServer.process(s, enc, seed=bytes(32)) for s in shards]

        device_process().close()  # warm-up at the measured shape
        for r in host_process():
            r.database.close()
        t0 = time.perf_counter()
        server = device_process()
        process_ms = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        host = host_process()
        host_process_ms = (time.perf_counter() - t0) * 1e3
        rows = np.bincount(server.databaseMap.chunkLocations[:, 0], minlength=SHARDS)
        for s, r in enumerate(host):
            assert np.array_equal(r.hint, server.hints[s])
            r.database.close()
        process_launches = launches(lambda: device_process().close())
        host_launches = launches(lambda: [r.database.close() for r in host_process()])
        chunks = len(server.databaseMap.chunkLocations)
        print(json.dumps({
            "shape": label, "card": name, "what": "process", "shards": SHARDS, "chunkSize": chunk,
            "rows": [int(r) for r in rows], "process_shards_ms": round(process_ms, 1),
            "host_shard_plus_process_ms": round(host_process_ms, 1),
            "process_shards_pcie_bytes": int(entries.nbytes + 8 * (count + 1) + 16 * chunks + 32 * SHARDS),
            "host_path_pcie_bytes": int(chunks * chunk + 32 * SHARDS),
            "process_shards_launches": process_launches, "host_path_launches": host_launches,
            "hints_equal": True}), flush=True)

        prm = server.params
        m = [p.columnSize for p in prm]
        k = [p.databaseColumns for p in prm]
        cpe = [p.chunksPerEntry for p in prm]
        singles = [sp.SimplePirServer(db, h, p) for db, h, p in zip(server.databases, server.hints, prm)]
        db4 = [db.export()[:4].astype(np.uint64) for db in server.databases]
        in_words, out_words = sum(c * kk for c, kk in zip(cpe, k)), sum(c * mm for c, mm in zip(cpe, m))
        for clients in [int(x) for x in args.clients.split(",")]:
            gen = torch.Generator(device="cuda").manual_seed(clients)
            per_shard = [torch.randint(0, 1 << 42, (clients, c, kk), device="cuda", dtype=torch.int64, generator=gen)
                         for c, kk in zip(cpe, k)]
            flat = torch.cat([q.reshape(clients, -1) for q in per_shard], dim=1).contiguous()
            d_out = torch.empty((clients, out_words), dtype=torch.int64, device="cuda")
            d_single = [torch.empty((clients, c, mm), dtype=torch.int64, device="cuda") for c, mm in zip(cpe, m)]
            stream = torch.cuda.current_stream().cuda_stream

            def grouped():
                server.computeResponsesDevice(flat.data_ptr(), 1, clients, d_out.data_ptr(), stream)

            def serial():
                for s in range(SHARDS):
                    singles[s].computeResponsesDevice(per_shard[s].data_ptr(), clients, d_single[s].data_ptr(), stream)

            grouped()
            serial()
            torch.cuda.synchronize()
            row = {"shape": label, "card": name, "what": "response", "clients": clients, "M": m, "K": k,
                   "chunksPerEntry": cpe,
                   "grouped_device_ms": median_event_ms(torch, grouped, args.reps),
                   "serial_device_ms": median_event_ms(torch, serial, args.reps),
                   "grouped_launches": launches(lambda: (grouped(), torch.cuda.synchronize())),
                   "serial_launches": launches(lambda: (serial(), torch.cuda.synchronize()))}
            out = d_out.cpu().numpy().view(np.uint64)
            at = 0
            for s in range(SHARDS):
                single = d_single[s].cpu().numpy().view(np.uint64)
                width = cpe[s] * m[s]
                for c in (0, clients - 1):
                    assert np.array_equal(out[c, at:at + width], single[c].reshape(-1)), (s, c)
                req0 = per_shard[s][0].cpu().numpy().view(np.uint64)
                got = out[0, at:at + width].reshape(cpe[s], m[s])[:, :4]
                assert np.array_equal(got, osp.response(db4[s], req0, 42))
                at += width
            if clients * in_words * 8 <= HOST_LIMIT:
                h_flat = flat.cpu().numpy().view(np.uint64)
                h_single = [q.cpu().numpy().view(np.uint64) for q in per_shard]
                row["grouped_host_ms"] = median_ms(lambda: server.computeResponses(h_flat, requests_per_shard=1),
                                                   args.reps)
                row["serial_host_ms"] = median_ms(lambda: [singles[s].computeResponses(h_single[s])
                                                           for s in range(SHARDS)], args.reps)
            else:
                row["grouped_host_ms"] = row["serial_host_ms"] = None
            row["parity"] = "ok"
            print(json.dumps(row), flush=True)
            del per_shard, flat, d_out, d_single
        server.close()


if __name__ == "__main__":
    main()
