"""SimplePIR server on the device (hecuda.simple_pir): processing and response times at the two shapes of DESIGN.md
section 6, N = 2048, errorStdDev 6.4, pt = 14, ct = 42 (the quantum128 bound):

  A  2^20 entries x 256 B     M = 147,    K = 1 048 576
  B  4096 entries x 256 KiB   M = 24 967, K = 24 576, chunksPerEntry 6

One JSON line per shape with process_ms (pack + hint, one call), the response's median call time at 1, 16 and 256
requests through the host-pointer call (response_ms) and the device-pointer call (device_ms, CUDA events), achieved
bytes/s of one database pass at 1 request and int8 op/s at 256 requests (2 x live digit pairs x M x K x queries; at
pt = 14 / ct = 42 the kernel runs 11 of the 12 pairs, the pair whose shift 8 (1 + 5) reaches ct adds nothing mod 2^ct),
and a parity check of the first 4 DB' rows of the first response against the oracle at every batch size.  process_ms
is one call after a warm-up call at the same shape; it covers the upload, the pack and the hint together.  The card's name and power limit are read in the same run."""
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

SHAPES = {"A": (1 << 20, 256), "B": (4096, 256 * 1024)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="A,B")
    ap.add_argument("--batches", default="1,16,256")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    hecuda.set_device(0)
    name = card()
    enc = sp.SimplePirEncryptionParams(14, 42, 2048, 6.4)
    for label in args.shapes.split(","):
        count, size = SHAPES[label]
        rng = np.random.default_rng(1)
        entries = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
        sp.SimplePirServer.process(entries, enc, seed=bytes(32)).database.close()  # warm-up at the measured shape
        t0 = time.perf_counter()
        res = sp.SimplePirServer.process(entries, enc, seed=bytes(32))
        process_ms = (time.perf_counter() - t0) * 1e3
        prm = res.params
        server = sp.SimplePirServer(res.database, res.hint, prm)
        m, k, cpe = prm.columnSize, prm.databaseColumns, prm.chunksPerEntry
        pairs = sum(1 for i in range(2) for j in range(6) if 8 * (i + j) < 42)
        db = res.database.export()[:4].astype(np.uint64)
        row = {"shape": label, "card": name, "M": m, "K": k, "chunksPerEntry": cpe, "process_ms": round(process_ms, 1)}
        for b in [int(x) for x in args.batches.split(",")]:
            reqs = rng.integers(0, 1 << 42, size=(b, cpe, k), dtype=np.uint64)
            server.computeResponses(reqs)
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                out = server.computeResponses(reqs)
                times.append((time.perf_counter() - t0) * 1e3)
            d_req = torch.from_numpy(reqs.view(np.int64)).cuda()
            d_out = torch.empty((b, cpe, m), dtype=torch.int64, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream
            server.computeResponsesDevice(d_req.data_ptr(), b, d_out.data_ptr(), stream)
            dev = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                server.computeResponsesDevice(d_req.data_ptr(), b, d_out.data_ptr(), stream)
                e1.record()
                torch.cuda.synchronize()
                dev.append(e0.elapsed_time(e1))
            row[f"response_ms_{b}"] = round(statistics.median(times), 3)
            row[f"device_ms_{b}"] = round(statistics.median(dev), 3)
            if b == 1:
                row["db_bytes_per_s_1"] = 2 * m * k / (statistics.median(dev) * 1e-3)
            if b == 256:
                row["int8_ops_per_s_256"] = 2 * pairs * m * k * b * cpe / (statistics.median(dev) * 1e-3)
            assert np.array_equal(out[0][:, :4], osp.response(db, reqs[0], 42)[:, :4])  # parity on 4 DB' rows
            del d_req, d_out
        row["parity"] = "ok"
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
