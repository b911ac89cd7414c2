"""Symmetric-PIR OPRF client rates on the device (hecuda.symmetric_pir.OprfClient's three calls, one thread per query):

  blind     hecuda_oprf_blind: queryContext(at:), Ser(r HashToGroup(keyword))
  finalize  hecuda_oprf_finalize: parse(oprfResponse:with:), VerifyProof, r^-1 D and Finalize's hash
  open      hecuda_symmetric_pir_open: decrypt(encryptedEntry:with:), AES-GCM-192 open

Keywords are "keyword <i mod 1024>", blinds random in [1, n - 1], responses made by hecuda_oprf_blind_evaluate (one
device call per batch) and entries sealed by symmetricPIRProcess at 64-byte values, each repeated to the batch size
(every query costs the same whatever its point).  One JSON line per (step, batch size), batches 1, 1024, 65536 and
1 000 000 by default, with:
  - call_ms / queries_per_s: wall time of one C-ABI call (uploads, kernels, downloads), `reps` runs after one warm-up,
    median reported;
  - kernels_ms / kernel_queries_per_s: each kernel of one call from torch.profiler, in a separate pass;
  - pcie_bytes: host-to-device and device-to-host bytes of one call, computed from the shapes;
then one line with the end-to-end chain blind -> OprfServer -> finalize at the largest batch (wall time of each call),
and one line with the Python restatement's rate (tests/oprf_proof_ref.py, one core), a CPU lower bound of seven P-384
ECDH scalar multiplications per finalize through cryptography (OpenSSL) on every host core, and a parity check of
sampled queries and outputs of the largest batch against the restatement.  Every line names the card and its power
limit, read in the same run."""
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
from hecuda import symmetric_pir as sp  # noqa: E402

KERNELS = {"blind": ("blind_kernel",), "finalize": ("verify_kernel", "unblind_kernel"), "open": ("open_kernel",)}
ECDH_PER_FINALIZE = 7  # d0 B, d0 D, s G, c pkS, s M, c Z, r^-1 D
DISTINCT, VALUE_BYTES = 1024, 64


def concatenate(blobs):
    offsets = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    return np.frombuffer(b"".join(blobs), dtype=np.uint8), offsets


def timed(call, reps):
    call()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()  # returns after its device-to-host copies
        times.append(time.perf_counter() - t0)
    return times, sorted(times)[len(times) // 2]


def kernel_times(call, names):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    kernels = dict.fromkeys(names, 0.0)
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        for name in names:
            if name in ev.key:
                kernels[name] += t / 1e3
    return kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,1024,65536,1000000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-queries", type=int, default=4)
    ap.add_argument("--parity-samples", type=int, default=6)
    ap.add_argument("--ecdh-per-core", type=int, default=500)
    args = ap.parse_args()
    if hecuda.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    hecuda.set_device(0)
    lib = hecuda.load_library()
    gpu = card()
    p = hecuda._ptr
    rng = random.Random(6)
    key = rng.randrange(1, sp.P384_ORDER).to_bytes(48, "big")
    config = sp.SymmetricPirConfig(key)
    pk = np.frombuffer(config.clientConfig().serverPublicKey, dtype=np.uint8)
    seed = np.frombuffer(bytes(range(32)), dtype=np.uint8)
    keywords = [b"keyword %d" % i for i in range(DISTINCT)]
    blinds = [rng.randrange(1, sp.P384_ORDER) for _ in keywords]
    contexts = sp.OprfClient(config.clientConfig()).queryContexts(keywords, blinds)
    base_queries = np.frombuffer(b"".join(c.query for c in contexts), dtype=np.uint8).reshape(DISTINCT, 49)
    base_blinds = np.frombuffer(b"".join(r.to_bytes(48, "big") for r in blinds), dtype=np.uint8).reshape(DISTINCT, 48)
    base_responses = np.frombuffer(b"".join(sp.OprfServer(config).computeResponses([c.query for c in contexts],
                                                                                   seed.tobytes())),
                                   dtype=np.uint8).reshape(DISTINCT, 145)
    rows = [(k, rng.randbytes(VALUE_BYTES)) for k in keywords]
    base_sealed = [v for _, v in sp.symmetricPIRProcess(rows, config)]
    base_outputs = np.stack([np.frombuffer(bytes(h), dtype=np.uint8) for h in sp.Oprf.evaluate(key, keywords)])

    last = None
    for n in [int(b) for b in args.batches.split(",")]:
        pick = np.arange(n) % DISTINCT
        data, offsets = concatenate([keywords[i] for i in pick])
        bl = np.ascontiguousarray(base_blinds[pick])
        queries = np.empty((n, 49), dtype=np.uint8)
        responses = np.ascontiguousarray(base_responses[pick])
        outputs = np.empty((n, 48), dtype=np.uint8)
        status = np.empty(n, dtype=np.uint8)
        sealed, sealed_offsets = concatenate([base_sealed[i] for i in pick])
        h = np.ascontiguousarray(base_outputs[pick])
        values = np.empty(max(sealed.size, 1), dtype=np.uint8)
        calls = {
            "blind": (lambda: hecuda._check(lib.hecuda_oprf_blind(p(data), p(offsets), n, p(bl), p(queries), p(status))),
                      data.nbytes + offsets.nbytes + bl.nbytes, queries.nbytes + status.nbytes),
            "finalize": (lambda: hecuda._check(lib.hecuda_oprf_finalize(p(pk), p(data), p(offsets), n, p(bl), p(queries),
                                                                        p(responses), p(outputs), p(status))),
                         data.nbytes + offsets.nbytes + bl.nbytes + queries.nbytes + responses.nbytes,
                         outputs.nbytes + status.nbytes),
            "open": (lambda: hecuda._check(lib.hecuda_symmetric_pir_open(p(h), p(sealed), p(sealed_offsets), n,
                                                                         p(values), p(status))),
                     h.nbytes + sealed.nbytes + sealed_offsets.nbytes + 256 + 1024, values.nbytes + status.nbytes),
        }
        for step, (call, h2d, d2h) in calls.items():
            times, median = timed(call, args.reps)
            assert int(status.sum()) == 0, f"{step}: a valid query was rejected"
            kernels = kernel_times(call, KERNELS[step])
            total = sum(kernels.values())
            print(json.dumps(dict(gpu, step=step, batch=n, call_ms=[round(t * 1e3, 2) for t in times],
                                  queries_per_s=round(n / median), kernels_ms={k: round(v, 3) for k, v in kernels.items()},
                                  kernel_queries_per_s=round(n / (total / 1e3)) if total else None,
                                  pcie_bytes={"h2d": int(h2d), "d2h": int(d2h)})), flush=True)
        assert np.array_equal(queries, base_queries[pick]) and np.array_equal(outputs, h)
        assert bytes(values[:VALUE_BYTES]) == rows[0][1]
        last = (n, pick, queries, outputs)

    # the chain blind -> OprfServer -> finalize at the largest batch, through the Python classes
    n, pick, _, _ = last
    client, server = sp.OprfClient(config.clientConfig()), sp.OprfServer(config)
    chain_keywords = [keywords[i] for i in pick]
    t0 = time.perf_counter()
    chain_contexts = client.queryContexts(chain_keywords, [blinds[i] for i in pick])
    t1 = time.perf_counter()
    chain_responses = server.computeResponses([c.query for c in chain_contexts], seed.tobytes())
    t2 = time.perf_counter()
    parsed = client.parseMany(chain_responses, chain_contexts)
    t3 = time.perf_counter()
    chain_ok = all(parsed[i] is not None and parsed[i].secretKey == bytes(base_outputs[pick[i]][24:])
                   for i in range(0, n, max(1, n // 1000)))
    print(json.dumps(dict(gpu, chain_batch=n, blind_s=round(t1 - t0, 3), server_s=round(t2 - t1, 3),
                          finalize_s=round(t3 - t2, 3), chain_queries_per_s=round(n / (t3 - t0)), chain_ok=chain_ok)),
          flush=True)

    import oprf_proof_ref as R
    n, pick, queries, outputs = last
    samples = sorted({0, n - 1} | {rng.randrange(n) for _ in range(args.parity_samples)})
    pk_bytes = pk.tobytes()
    parity = all(
        queries[i].tobytes() == R.OprfClient(pk_bytes).queryContext(keywords[pick[i]], blinds[pick[i]])[2] and
        outputs[i].tobytes() == R.finalize_verifiable(keywords[pick[i]], blinds[pick[i]],
                                                      base_responses[pick[i]].tobytes(), pk_bytes)
        for i in samples)
    t0 = time.perf_counter()
    for i in range(args.oracle_queries):
        R.finalize_verifiable(keywords[i], blinds[i], base_responses[i].tobytes(), pk_bytes)
    oracle_rate = args.oracle_queries / (time.perf_counter() - t0)
    cores, ecdh_rate = cpu_ecdh_rate(args.ecdh_per_core)
    print(json.dumps(dict(gpu, parity_samples=len(samples), parity_ok=parity,
                          oracle_finalize_per_s=round(oracle_rate, 1), cpu_ecdh_per_s=round(ecdh_rate),
                          cpu_finalize_per_s_bound=round(ecdh_rate / ECDH_PER_FINALIZE), cpu_cores=cores,
                          cpu_note="lower bound: seven P-384 ECDH scalar multiplies per finalize "
                                   "(cryptography/OpenSSL), all host cores; no hashing")))
    if not (parity and chain_ok):
        raise SystemExit("parity check failed")


if __name__ == "__main__":
    main()
