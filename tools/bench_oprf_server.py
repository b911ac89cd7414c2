"""Symmetric-PIR OPRF server rate (hecuda_oprf_blind_evaluate: OprfServer.computeResponse on the device, RFC 9497
BlindEvaluate with the DLEQ proof, one thread per query).

Queries are valid compressed P-384 points made by cryptography from seeded keys: 1024 distinct points, repeated to the
batch size (every query costs the same whatever its point).  One JSON line per batch size (default 1, 1024, 65536 and
1 000 000) with:
  - call_ms / queries_per_s: wall time of one C-ABI call (uploads, kernels, downloads), `reps` runs after one warm-up,
    median reported;
  - kernels_ms / kernel_queries_per_s: each kernel of one call from torch.profiler, in a separate pass;
  - pcie_bytes: host-to-device and device-to-host bytes of one call, computed from the shape;
then one line with the oracle's rate (tests/oprf_proof_ref.py, Python integers, one core), a CPU lower bound of five
P-384 ECDH scalar multiplications per query through cryptography (OpenSSL) on every host core, and a parity check of
sampled responses of the largest batch against the oracle.  Every line names the card and its power limit, read in
the same run."""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tools"),
                os.path.join(ROOT, "tests")]

import hecuda  # noqa: E402
from bench_symmetric_pir import card, cpu_ecdh_rate  # noqa: E402

KERNELS = ("proof_setup_kernel", "blind_evaluate_kernel", "proof_kernel")
ECDH_PER_QUERY = 5


def distinct_points(count):
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric import ec

    rng = random.Random(4)
    return [ec.derive_private_key(rng.randrange(1, 2**383), ec.SECP384R1()).public_key().public_bytes(
        serialization.Encoding.X962, serialization.PublicFormat.CompressedPoint) for _ in range(count)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,1024,65536,1000000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-queries", type=int, default=10)
    ap.add_argument("--parity-samples", type=int, default=8)
    ap.add_argument("--ecdh-per-core", type=int, default=500)
    args = ap.parse_args()
    if hecuda.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    hecuda.set_device(0)
    lib = hecuda.load_library()
    gpu = card()
    key_bytes = random.Random(2).randrange(1, 2**383).to_bytes(48, "big")
    key = np.frombuffer(key_bytes, dtype=np.uint8)
    seed = np.frombuffer(bytes(range(32)), dtype=np.uint8)
    points = np.frombuffer(b"".join(distinct_points(1024)), dtype=np.uint8).reshape(1024, 49)
    p = hecuda._ptr
    from torch.profiler import ProfilerActivity, profile

    last = None
    for n in [int(b) for b in args.batches.split(",")]:
        queries = np.ascontiguousarray(points[np.arange(n) % len(points)])
        responses = np.empty((n, 145), dtype=np.uint8)
        status = np.empty(n, dtype=np.uint8)

        def call():
            hecuda._check(lib.hecuda_oprf_blind_evaluate(p(key), p(queries), n, p(seed), p(responses), p(status)))

        call()
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            call()  # returns after its device-to-host copies
            times.append(time.perf_counter() - t0)
        median = sorted(times)[len(times) // 2]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        kernels = dict.fromkeys(KERNELS, 0.0)
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            for name in KERNELS:
                if name in ev.key:
                    kernels[name] += t / 1e3
        total = sum(kernels.values())
        assert int(status.sum()) == 0, "a valid query was reported invalid"
        print(json.dumps(dict(gpu, batch=n, call_ms=[round(t * 1e3, 2) for t in times], queries_per_s=round(n / median),
                              kernels_ms={k: round(v, 3) for k, v in kernels.items()},
                              kernel_queries_per_s=round(n / (total / 1e3)) if total else None,
                              pcie_bytes={"h2d": queries.nbytes + seed.nbytes + 97 + 48,
                                          "d2h": responses.nbytes + status.nbytes})), flush=True)
        last = (queries, responses)

    import oprf_proof_ref as R
    queries, responses = last
    rng = random.Random(5)
    samples = sorted({0, len(queries) - 1} | {rng.randrange(len(queries)) for _ in range(args.parity_samples)})
    parity = all(responses[i].tobytes() == R.blind_evaluate_verifiable(key_bytes, queries[i].tobytes(), seed.tobytes())
                 for i in samples)
    t0 = time.perf_counter()
    for i in range(args.oracle_queries):
        R.blind_evaluate_verifiable(key_bytes, points[i].tobytes(), seed.tobytes())
    oracle_rate = args.oracle_queries / (time.perf_counter() - t0)
    cores, ecdh_rate = cpu_ecdh_rate(args.ecdh_per_core)
    print(json.dumps(dict(gpu, parity_samples=len(samples), parity_ok=parity, oracle_queries_per_s=round(oracle_rate, 1),
                          cpu_ecdh_per_s=round(ecdh_rate), cpu_queries_per_s_bound=round(ecdh_rate / ECDH_PER_QUERY),
                          cpu_cores=cores,
                          cpu_note="lower bound: five P-384 ECDH scalar multiplies per query (cryptography/OpenSSL), "
                                   "all host cores; no hashing, no proof")))
    if not parity:
        raise SystemExit("parity check failed")


if __name__ == "__main__":
    main()
