"""The PNNS client and float database processing on the device, at the C5 shape (N = 8192, 4 x 55-bit moduli, t = 65537,
512-dimensional vectors, 16 query vectors), with and without one extra 17-bit plaintext modulus.

Rows, one JSON line each:
  - queries_per_s: Client.generateQuery of 16 float vectors (hecuda_pnns_query_generate per context), full and seeded;
  - distance_matrices_per_s: Client.decrypt of one response (hecuda_pnns_decrypt_distances) for the database rows x 16;
  - process_from_floats_s against process_from_int64_s: ProcessedDatabase.processOnDevice from float rows, and
    PlaintextMatrix.fromSignedValues from host int64 values already rounded (one per context), wall time and the bytes
    each sends over PCIe;
  - validate_s: ProcessedDatabase.validate(16 query vectors, trials=1).
`reps` timed runs follow one warm-up; the median is reported.  The first line names the card and its power limit."""
import argparse
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tools")]

import hecuda  # noqa: E402
from hecuda import pnns  # noqa: E402
from bench_client import card, emit, timed  # noqa: E402

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]
N, T, DIM, QUERIES = 8192, 65537, 512, 16
EXTRA_T = 114689  # 7 * 2^14 + 1, the next 17-bit prime = 1 mod 2N


def run(rows, reps, extra):
    ts = [T] + ([EXTRA_T] if extra else [])
    label = f"C5 rows={rows} moduli={len(ts)}"
    ctxs = [hecuda.Context(N, Q8192, t) for t in ts]
    s = pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, DIM, ts)
    ekc = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(rows, DIM), QUERIES, N)
    cc = pnns.ClientConfig(pnns.EncryptionParameters(N, T, tuple(Q8192)), s, DIM, ekc, extraPlaintextModuli=ts[1:])
    sc = pnns.ServerConfig(cc)
    rng = np.random.default_rng(7)
    vectors = rng.standard_normal((rows, DIM)).astype(np.float32)
    db = pnns.Database([pnns.DatabaseRow(i, b"", v) for i, v in enumerate(vectors)])

    def from_floats():
        pnns.ProcessedDatabase.processOnDevice(db, sc, ctxs).close()

    emit(context=label, op="process_from_floats_s", value=timed(from_floats, reps), pcie_bytes=vectors.nbytes)
    values = np.ascontiguousarray(np.rint(vectors * 10).astype(np.int64))   # stands in for values rounded on the host

    def from_int64():
        for ctx in ctxs:
            pnns.PlaintextMatrix.fromSignedValues(ctx, pnns.MatrixDimensions(rows, DIM), values % ctx.plaintextModulus,
                                                  sc.babyStepGiantStep, reduce=True).close()

    emit(context=label, op="process_from_int64_s", value=timed(from_int64, reps), pcie_bytes=values.nbytes * len(ctxs))

    processed = pnns.ProcessedDatabase.processOnDevice(db, sc, ctxs)
    client, server = pnns.Client(cc, ctxs), pnns.Server(processed)
    sk = client.generateSecretKey()
    key = client.generateEvaluationKey(sk)
    queries = vectors[:QUERIES]
    emit(context=label, op="queries_per_s", batch=QUERIES, value=1 / timed(lambda: client.generateQuery(queries, sk), reps))
    emit(context=label, op="seeded_queries_per_s", batch=QUERIES,
         value=1 / timed(lambda: client.generateQuery(queries, sk, wire=True), reps))
    response = server.computeResponse(client.generateQuery(queries, sk), key)
    emit(context=label, op="distance_matrices_per_s", shape=[rows, QUERIES],
         value=1 / timed(lambda: client.decrypt(response, sk), reps))
    times = []
    for _ in range(reps + 1):
        start = time.perf_counter()
        processed.validate(queries, trials=1).evaluationKey.close()
        times.append(time.perf_counter() - start)
    emit(context=label, op="validate_s", value=statistics.median(times[1:]))
    key.close()
    processed.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    emit(**card())
    for extra in (False, True):
        run(args.rows, args.reps, extra)


if __name__ == "__main__":
    main()
