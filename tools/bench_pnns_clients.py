#!/usr/bin/env python
"""PNNS with one-vector clients, each with its own evaluation key, at the BASELINE config 5 shape (100 000 x 512 matrix,
N = 8192, four 55-bit moduli): K clients answered (a) by K single-client hecuda_pnns_mul_transpose_matrix calls,
(b) by one hecuda_pnns_compute_response_clients call, (c) by one hecuda_pnns_compute_response_clients_wire call.

    python tools/bench_pnns_clients.py [K ...]        (default K = 1 4 16 64)

Synthetic: uniform coefficient plaintexts < t for the matrix, uniform residues for every client's Galois keys and query
ciphertext, uniform seeds.  Warms every call shape up, then runs two rounds that alternate (a), (b), (c).  Prints one
JSON line: clients/s per round, kernel launches and PCIe bytes per client, the card and its power limit (read in the
same run), and whether every client's (b) reply equals its (a) reply.
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")):
    sys.path.insert(0, p)
import numpy as np

import hecuda
from hecuda import pnns
from hecuda.pir import skipLSBsForDecryption

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]


def uniform(rng, moduli, prefix, n):
    out = np.empty(tuple(prefix) + (len(moduli), n), dtype=np.uint64)
    for i, q in enumerate(moduli):
        out[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (n,), dtype=np.uint64)
    return out


def card():
    """Name and power limit of the GPU, read-only."""
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in line.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as exc:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(exc)}


def run(counts=(1, 4, 16, 64), rows=100000, dim=512, rounds=2):
    n, t = 8192, 65537
    if hecuda.device_count() < 1:
        raise RuntimeError("bench_pnns_clients needs a CUDA device")
    ctx = hecuda.Context(n, Q8192, t)
    L = ctx.L
    rng = np.random.default_rng(8)
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(dim)
    results = -(-rows // n)
    plain = rng.integers(0, t, size=(bsgs.vectorDimension * results, n), dtype=np.uint64)
    matrix = pnns.PlaintextMatrix(ctx, pnns.MatrixDimensions(rows, dim), None, bsgs, plaintexts=plain)
    del plain
    dims = pnns.MatrixDimensions(1, dim)
    elements = {pnns.GaloisElement.rotatingColumns(-1, n), pnns.GaloisElement.rotatingColumns(-bsgs.babyStep, n)}
    top = max(counts)
    keys = []
    for _ in range(top):
        key = hecuda.EvaluationKey(ctx, None)
        for e in elements:
            key.setGaloisKey(e, uniform(rng, Q8192, (L, 2), n))
        keys.append(key)
    cts = uniform(rng, Q8192[:L], (top, 1, 2), n)                     # one query ciphertext per client, Coeff
    poly0 = hecuda.Bfv.serialize(ctx, cts[:, 0, 0]).reshape(top, 1, -1)  # .seeded: poly0 and a seed per ciphertext
    seeds = rng.integers(0, 256, size=(top, 1, 32), dtype=np.uint8)
    skips = skipLSBsForDecryption(ctx)
    reply_bytes = sum(hecuda.Bfv.serializationByteCount(ctx, 1, s) for s in skips)

    def single(k):
        return [matrix.mulTransposeMatrix(cts[j], dims, keys[j], modSwitchDownToSingle=True) for j in range(k)]

    def clients(k):
        return matrix.computeResponses(cts[:k], dims, keys[:k])

    def wire(k):
        return pnns.PnnsWire.computeResponses(matrix, poly0[:k], seeds[:k], dims, keys[:k])[0]

    def timed(fn, k):
        before = hecuda.kernel_launch_count()
        t0 = time.perf_counter()
        out = fn(k)  # every call returns after its stream has drained
        return time.perf_counter() - t0, hecuda.kernel_launch_count() - before, out

    out = {"metric": "PNNS clients/s, one query vector and one evaluation key per client (matrix resident in HBM)",
           "config": {"workload": f"N={n}, 4 x 55-bit moduli, t={t}, matrix {rows} x {dim}, babyStep={bsgs.babyStep}, "
                                  f"giantStep={bsgs.giantStep}, replies/client={results}"},
           **card(), "rounds": rounds, "runs": []}
    ct_bytes = 2 * L * n * 8
    for k in counts:
        for fn in (single, clients, wire):  # warm-up: every shape the timed rounds use
            fn(k)
        secs = {"a": [], "b": [], "c": []}
        launches = {}
        same = True
        for _ in range(rounds):
            for name, fn in (("a", single), ("b", clients), ("c", wire)):
                s, lc, got = timed(fn, k)
                secs[name].append(s)
                launches[name] = lc
                if name == "a":
                    want = got
                elif name == "b":
                    same = same and all(np.array_equal(got[j], want[j]) for j in range(k))
        run_out = {"clients": k}
        for name, label in (("a", "single_calls"), ("b", "clients_call"), ("c", "clients_wire_call")):
            run_out[label] = {"clients_per_s": [round(k / s, 2) for s in secs[name]],
                              "launches_per_client": round(launches[name] / k, 1)}
        run_out["single_calls"]["pcie_bytes_per_client"] = {"h2d": ct_bytes, "d2h": results * 2 * n * 8}
        run_out["clients_call"]["pcie_bytes_per_client"] = {"h2d": ct_bytes, "d2h": results * 2 * n * 8}
        run_out["clients_wire_call"]["pcie_bytes_per_client"] = {"h2d": int(poly0.shape[2]) + 32, "d2h": results * reply_bytes}
        run_out["clients_call_equals_single_calls"] = bool(same)
        run_out["speedup_b_over_a"] = round(min(secs["a"]) / min(secs["b"]), 3)
        out["runs"].append(run_out)
    for key in keys:
        key.close()
    matrix.close()
    ctx.close()
    return out


def main():
    counts = tuple(int(a) for a in sys.argv[1:]) or (1, 4, 16, 64)
    print(json.dumps(run(counts)))


if __name__ == "__main__":
    main()
