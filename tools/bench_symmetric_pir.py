"""Symmetric keyword PIR processing rate (hecuda_symmetric_pir_process: KeywordDatabase.symmetricPIRProcess on the
device, P-384 OPRF and AES-GCM-192 per row).

Shape (synthetic, seeded): --rows rows (default 1 000 000) with 12-byte keywords and 64-byte values.  One JSON line
with:
  - process_ms / rows_per_s: wall time of one C-ABI call (uploads, OPRF kernels, seal kernels, downloads), `reps` runs
    after one warm-up, median reported;
  - kernels_ms: the OPRF and seal kernels of one call from torch.profiler, in a separate pass;
  - pcie_bytes: host-to-device and device-to-host bytes of one call, computed from the shape;
  - oracle_rows_per_s: oracle/oprf_oracle.py (Python integers) on one core, for scale;
  - cpu_ecdh_rows_per_s: a CPU lower bound: one P-384 ECDH scalar multiplication per row through cryptography (OpenSSL)
    on every host core.  Scalar multiply only: no hash-to-curve, no hashing, no sealing.
The line names the card and its power limit, read in the same run."""
import argparse
import concurrent.futures
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")]

import hecuda  # noqa: E402

KEYWORD_BYTES, VALUE_BYTES = 12, 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "error": str(e)}


def ecdh_rows(count):
    from cryptography.hazmat.primitives.asymmetric import ec

    key = ec.generate_private_key(ec.SECP384R1())
    peer = ec.generate_private_key(ec.SECP384R1()).public_key()
    t0 = time.perf_counter()
    for _ in range(count):
        key.exchange(ec.ECDH(), peer)
    return count, time.perf_counter() - t0


def cpu_ecdh_rate(rows_per_core):
    cores = os.cpu_count() or 1
    with concurrent.futures.ProcessPoolExecutor(cores) as pool:
        ecdh_rows(10)
        t0 = time.perf_counter()
        done = sum(n for n, _ in pool.map(ecdh_rows, [rows_per_core] * cores))
        return cores, done / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-rows", type=int, default=50)
    ap.add_argument("--ecdh-rows-per-core", type=int, default=500)
    args = ap.parse_args()
    if hecuda.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    hecuda.set_device(0)
    lib = hecuda.load_library()
    n = args.rows
    rng = np.random.default_rng(1)
    key = np.frombuffer(random.Random(2).randrange(1, 2**383).to_bytes(48, "big"), dtype=np.uint8)
    keywords = rng.integers(0, 256, n * KEYWORD_BYTES, dtype=np.uint8)
    values = rng.integers(0, 256, n * VALUE_BYTES, dtype=np.uint8)
    koff = np.arange(n + 1, dtype=np.uint64) * KEYWORD_BYTES
    voff = np.arange(n + 1, dtype=np.uint64) * VALUE_BYTES
    kout = np.empty(16 * n, dtype=np.uint8)
    vout = np.empty((VALUE_BYTES + 16) * n, dtype=np.uint8)
    p = hecuda._ptr

    def call():
        hecuda._check(lib.hecuda_symmetric_pir_process(p(key), p(keywords), p(koff), p(values), p(voff), n, p(kout),
                                                       p(vout)))

    call()
    times = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        call()  # returns after its device-to-host copies
        times.append(time.perf_counter() - t0)
    median = sorted(times)[len(times) // 2]

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    kernels = {"oprf_evaluate_kernel": 0.0, "seal_kernel": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        for name in kernels:
            if name in ev.key:
                kernels[name] += t / 1e3

    from oracle import oprf_oracle as O
    orng = random.Random(3)
    t0 = time.perf_counter()
    for _ in range(args.oracle_rows):
        h = O.evaluate(key.tobytes(), orng.randbytes(KEYWORD_BYTES))
        O.seal(h, orng.randbytes(VALUE_BYTES))
    oracle_rate = args.oracle_rows / (time.perf_counter() - t0)
    cores, ecdh_rate = cpu_ecdh_rate(args.ecdh_rows_per_core)

    h2d = keywords.nbytes + koff.nbytes + values.nbytes + voff.nbytes + 97
    d2h = kout.nbytes + vout.nbytes
    out = dict(card(), rows=n, keyword_bytes=KEYWORD_BYTES, value_bytes=VALUE_BYTES,
               process_ms=[round(t * 1e3, 1) for t in times], rows_per_s=round(n / median),
               kernels_ms={k: round(v, 3) for k, v in kernels.items()},
               kernel_rows_per_s=round(n / (sum(kernels.values()) / 1e3)) if sum(kernels.values()) else None,
               pcie_bytes={"h2d": h2d, "d2h": d2h}, oracle_rows_per_s=round(oracle_rate, 1),
               cpu_ecdh_rows_per_s=round(ecdh_rate), cpu_cores=cores,
               cpu_note="lower bound: one P-384 ECDH scalar multiply per row (cryptography/OpenSSL), all host cores")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
