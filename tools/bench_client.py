"""Client-side throughput on the device (hecuda_bfv_generate_secret_key, hecuda_bfv_encrypt[_seeded], hecuda_evk_generate,
hecuda_bfv_noise_budget) and PIR shard validation wall time (KeywordPirServer.validate).

Rows, one JSON line each:
  - secret_keys_per_s, encryptions_per_s (full and seeded), noise_budgets_per_s: host-pointer C-ABI calls over a batch
    at N = 8192 with the C2 moduli (4 x 55 bits, t = 557057) and at N = 4096 with the PIR moduli (27/28/28 bits, t = 17);
  - evaluation_keys_per_s at the MulPir key configuration of a 100 000 x 2 B index database (N = 4096, relinearization
    + Galois keys) and at the C5 PNNS configuration (N = 8192, 4 x 55-bit moduli, the 512-dimension BSGS Galois keys);
  - validate_s: wall time of KeywordPirServer.validate(row, trials=1) per shard at the keyword shapes of DESIGN.md 6
    (100 000 x 2 B and 1 000 x 60 000 B at t = 17; 2^20 x 64 B with --large), the database processed beforehand;
  - oracle_*: the same operation in oracle/client_oracle.py (a Python restatement, not the reference) for scale.
`reps` timed runs follow one warm-up; the median is reported.  The first line names the card and its power limit."""
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
from hecuda import keyword_pir as kw  # noqa: E402
from hecuda import pir, pnns  # noqa: E402

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]
PIR_MODULI = [134176769, 268369921, 268361729]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "error": str(e)}


def timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        start = time.perf_counter()
        fn()
        times.append(time.perf_counter() - start)
    return statistics.median(times)


def emit(**row):
    print(json.dumps(row), flush=True)


def bench_context(name, n, moduli, t, batch, reps, oracle):
    g = hecuda.Context(n, moduli, t)
    lib = hecuda.load_library()
    K = len(moduli)
    seeds = np.frombuffer(os.urandom(32 * batch), dtype=np.uint8).reshape(batch, 32).copy()
    keys = np.empty((batch, K, n), dtype=np.uint64)
    s = timed(lambda: lib.hecuda_bfv_generate_secret_key(g._h, hecuda._ptr(seeds), hecuda._ptr(keys), batch), reps)
    emit(context=name, op="secret_keys_per_s", batch=batch, value=batch / s)
    sk = hecuda.SecretKey.generate(g)
    pts = np.random.default_rng(1).integers(0, t, size=(batch, n), dtype=np.uint64)
    s = timed(lambda: hecuda.Bfv.encrypt(g, sk, pts), reps)
    emit(context=name, op="encryptions_per_s", batch=batch, value=batch / s)
    s = timed(lambda: hecuda.Bfv.encrypt(g, sk, pts, seeded=True), reps)
    emit(context=name, op="seeded_encryptions_per_s", batch=batch, value=batch / s)
    cts = hecuda.Bfv.encrypt(g, sk, pts)
    s = timed(lambda: hecuda.Bfv.noiseBudget(g, sk, cts), reps)
    emit(context=name, op="noise_budgets_per_s", batch=batch, value=batch / s)
    if oracle:
        from oracle import client_oracle as co
        start = time.perf_counter()
        co.encrypt(n, moduli[:g.L], t, sk.poly, pts[0], os.urandom(32), os.urandom(32))
        emit(context=name, op="oracle_encryptions_per_s", batch=1, value=1 / (time.perf_counter() - start))
        start = time.perf_counter()
        co.noise_budget(n, moduli, t, sk.poly, cts[0])
        emit(context=name, op="oracle_noise_budgets_per_s", batch=1, value=1 / (time.perf_counter() - start))
    g.close()


def bench_evk(name, n, moduli, t, config, reps, oracle):
    g = hecuda.Context(n, moduli, t)
    sk = hecuda.SecretKey.generate(g)

    def one():
        hecuda.EvaluationKey.generate(g, config, sk).close()
    s = timed(one, reps)
    emit(context=name, op="evaluation_keys_per_s", galois_keys=len(config.galoisElements),
         relin=config.hasRelinearizationKey, value=1 / s)
    if oracle:
        from oracle import client_oracle as co
        L = g.L
        count = (int(config.hasRelinearizationKey) + len(config.galoisElements)) * L
        seeds = [os.urandom(32) for _ in range(count)]
        start = time.perf_counter()
        co.generate_evaluation_key(n, moduli[:L], moduli[L], sk.poly, config.hasRelinearizationKey,
                                   config.galoisElements, seeds, seeds)
        emit(context=name, op="oracle_evaluation_keys_per_s", value=1 / (time.perf_counter() - start))
    g.close()


def rows_for(count, size, seed):
    rng = np.random.default_rng(seed)
    keywords = rng.integers(0, 256, size=(count, 16), dtype=np.uint8)
    values = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
    return [(keywords[i].tobytes(), values[i].tobytes()) for i in range(count)]


def bench_validate(count, size, reps):
    g = hecuda.Context(4096, PIR_MODULI, 17)
    bpp = g.degree * (g.plaintextModulus.bit_length() - 1) // 8
    single = kw.serializedSize(size)
    bucket = -(-single // bpp) * bpp if single >= bpp // 2 else bpp // 2   # defaultMaxSerializedBucketSize
    config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(bucket), False, "hybridCompression")
    rows = rows_for(count, size, 7)
    processed = kw.KeywordPirServer.processOnDevice(rows, config, g)
    server = kw.KeywordPirServer(g, processed)
    budgets = []

    def one():
        result = server.validate(rows[count // 2], trials=1)
        budgets.append(result.noiseBudget)
        result.evaluationKey.close()
    s = timed(one, reps)
    emit(context="n4096_pir_t17", op="validate_s", shape=f"{count} x {size} B", dimensions=processed.pirParameter.dimensions,
         value=s, noise_budget=min(budgets))
    processed.close()
    g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--large", action="store_true", help="also validate the 2^20 x 64 B keyword shape")
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    hecuda.set_device(0)
    emit(**card())
    oracle = not args.no_oracle
    bench_context("n8192_c2", 8192, Q8192, 557057, args.batch, args.reps, oracle)
    bench_context("n4096_pir_t17", 4096, PIR_MODULI, 17, args.batch, args.reps, oracle)
    mulpir = pir.MulPir.generateParameter(pir.IndexPirConfig(100000, 2, 2, 2, False, "hybridCompression"),
                                          hecuda.Context(4096, PIR_MODULI, 17))
    bench_evk("mulpir_n4096_t17", 4096, PIR_MODULI, 17, mulpir.evaluationKeyConfig, args.reps, oracle)
    elements = [pnns.GaloisElement.rotatingColumns(-1, 8192)]
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(512)
    if bsgs.giantStep > 1:
        elements.append(pnns.GaloisElement.rotatingColumns(-bsgs.babyStep, 8192))
    bench_evk("c5_pnns_n8192", 8192, Q8192, 65537,
              pir.EvaluationKeyConfig(list(dict.fromkeys(elements)), False), args.reps, oracle)
    for count, size in [(100000, 2), (1000, 60000)] + ([(1 << 20, 64)] if args.large else []):
        bench_validate(count, size, max(1, args.reps // 2))


if __name__ == "__main__":
    main()
