#!/usr/bin/env python
"""Evaluation keys from the wire (hecuda_evk_create_serialized) and many clients' serialized MulPir queries in one call
(hecuda_mulpir_compute_response_clients_wire).

    python tools/bench_evk_wire.py [--reps R] [--clients K] [--entries N] [--skip-pir]

Reports, for one client's SerializedEvaluationKey (relinearization key + the Galois keys of the MulPir
EvaluationKeyConfig) at the PIR default parameters (N = 4096, q = 27/28/28 bits) and at N = 8192, 4 x 55 bits:
  - the wire load: keys/s, key ciphertexts/s and key bytes written/s (host call, copies in and the final synchronise
    included) against HBM's 3.35 TB/s, plus the two kernels' device time from torch.profiler in a separate pass;
  - the same keys loaded from prebuilt 64-bit words (hecuda_evk_create + hecuda_evk_set_galois_key);
and, at the C4 shape of tools/bench_pir.py (2^20 entries x 64 B, N = 4096), queries/s of K clients through the
many-clients wire call against the word-based many-clients call (host calls, copies included).  Prints one JSON line per
measurement, and the card's name and power limit read in the same run.  Key, query and database values are uniform
residues: what the server computes does not depend on them being well-formed."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200")):
    sys.path.insert(0, p)

import numpy as np
import torch

import hecuda
from hecuda import pir

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:357-367)
HBM_BYTES_PER_S = 3.35e12                       # H100 SXM data sheet
KEY_KERNELS = ("drbg_chain_kernel", "key_expand_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def uniform(rng, moduli, shape_prefix, n):
    out = np.empty(tuple(shape_prefix) + (len(moduli), n), dtype=np.uint64)
    for i, q in enumerate(moduli):
        out[..., i, :] = rng.integers(0, q, size=tuple(shape_prefix) + (n,), dtype=np.uint64)
    return out


def pir_setup(ctx, entries, entry_size, rng):
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(entries, entry_size, 2, 1, True, "hybridCompression", False), ctx)
    chunks = -(-param.encodedEntrySize // pir.bytesPerPlaintext(ctx))
    count = chunks * int(np.prod(param.dimensions))
    db = pir.ProcessedDatabase(ctx, rng.integers(0, ctx.plaintextModulus, size=(count, ctx.degree), dtype=np.uint64), None,
                               evalFormat=False)
    return param, pir.MulPirServer(param, ctx, [db])


def wire_key(ctx, rng, elements):
    """One client's key: words (relin, {e: key}) and the wire form of the same values."""
    L, n = ctx.L, ctx.degree
    moduli = ctx.coefficientModuli

    def one():
        words = uniform(rng, moduli, (L, 2), n)
        poly0 = hecuda.Bfv.serialize(ctx, words[:, 0], base=hecuda.BASE_KEYSWITCH)
        return words, (poly0, rng.integers(0, 256, size=(L, 32), dtype=np.uint8))

    relin = one()
    galois = {e: one() for e in elements}
    return relin, galois


def timed(fn, reps):
    fn()  # warm-up
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps


class KeyBench:
    """One client's key at one parameter set: wire and word loads."""

    def __init__(self, name, ctx, elements):
        self.name, self.ctx, self.elements = name, ctx, elements
        self.relin, self.galois = wire_key(ctx, np.random.default_rng(7), elements)
        L, n = ctx.L, ctx.degree
        self.cts = (1 + len(elements)) * L
        self.key_bytes = self.cts * 2 * (L + 1) * n * 8
        self.wire_bytes = sum(p.nbytes + s.nbytes for p, s in [self.relin[1]] + [g[1] for g in self.galois.values()])

    def load_wire(self):
        gw = {e: g[1] for e, g in self.galois.items()}
        hecuda.EvaluationKey.fromSerialized(self.ctx, self.relin[1][0], self.relin[1][1], gw).close()

    def load_words(self):
        k = hecuda.EvaluationKey(self.ctx, self.relin[0])
        for e, g in self.galois.items():
            k.setGaloisKey(e, g[0])
        k.close()

    def time(self, reps):
        wire_s, words_s = timed(self.load_wire, reps), timed(self.load_words, reps)
        return dict(measure="evk_load", shape=self.name, elements=len(self.elements), key_ciphertexts=self.cts,
                    key_bytes=self.key_bytes, wire_bytes=self.wire_bytes,
                    wire=dict(keys_per_s=1 / wire_s, key_ciphertexts_per_s=self.cts / wire_s,
                              bytes_written_per_s=self.key_bytes / wire_s,
                              share_of_hbm=self.key_bytes / wire_s / HBM_BYTES_PER_S),
                    words=dict(keys_per_s=1 / words_s, key_ciphertexts_per_s=self.cts / words_s))

    def kernels(self, reps):
        """Device time of the two kernels per key.  Run after every timing: the profiler slows later runtime calls."""
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                self.load_wire()
            torch.cuda.synchronize()
        kernel_us = {k: 0.0 for k in KEY_KERNELS}
        for ev in prof.key_averages():
            for k in KEY_KERNELS:
                if k in ev.key:
                    kernel_us[k] += ev.device_time_total / reps
        expand_s = kernel_us["key_expand_kernel"] * 1e-6
        return dict(measure="evk_kernels", shape=self.name, kernels_us=kernel_us,
                    expand_kernel_bytes_per_s=self.key_bytes / expand_s if expand_s else None,
                    expand_kernel_share_of_hbm=self.key_bytes / expand_s / HBM_BYTES_PER_S if expand_s else None)


def bench_clients(ctx, entries, k, reps):
    rng = np.random.default_rng(3)
    param, server = pir_setup(ctx, entries, 64, rng)
    elements = param.evaluationKeyConfig.galoisElements
    L, n = ctx.L, ctx.degree
    qct = -(-param.expandedQueryCount // n)
    keys, poly0, seeds = [], [], []
    for c in range(k):
        relin, galois = wire_key(ctx, np.random.default_rng(100 + c), elements)
        keys.append(hecuda.EvaluationKey.fromSerialized(ctx, relin[1][0], relin[1][1], {e: g[1] for e, g in galois.items()}))
        cts = uniform(rng, ctx.ciphertextModuli, (qct,), n)
        poly0.append(hecuda.Bfv.serialize(ctx, cts))
        seeds.append(rng.integers(0, 256, size=(qct, 32), dtype=np.uint8))
    poly0, seeds = np.stack(poly0), np.stack(seeds)
    # the word-based call takes the same queries expanded on the host side of the comparison (expandSeeded)
    words = np.stack([hecuda.Bfv.expandSeeded(ctx, poly0[c], seeds[c]) for c in range(k)])
    wire, _ = pir.PirWire.computeResponses(server, poly0, seeds, keys)
    single, _ = pir.PirWire.computeResponse(server, poly0[k - 1], seeds[k - 1], keys[k - 1])
    assert np.array_equal(wire[k - 1], single), "many-clients wire reply differs from the single-client wire call"
    wire_s = timed(lambda: pir.PirWire.computeResponses(server, poly0, seeds, keys), reps)
    words_s = timed(lambda: server.computeResponses(words, keys), reps)
    print(json.dumps(dict(measure="mulpir_clients", dims=param.dimensions, clients=k, query_ciphertexts=qct,
                          query_wire_bytes=int(poly0[0].nbytes + seeds[0].nbytes), query_word_bytes=int(words[0].nbytes),
                          wire_queries_per_s=k / wire_s, words_queries_per_s=k / words_s)), flush=True)
    for key in keys:
        key.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--clients", type=int, default=16)
    ap.add_argument("--entries", type=int, default=1 << 20)
    ap.add_argument("--skip-pir", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evk_wire needs a CUDA device")
    print(json.dumps(dict(card=card())), flush=True)
    from oracle import oracle as orc

    config = pir.IndexPirConfig(args.entries, 64, 2, 1, True, "hybridCompression", False)
    pir_ctx = hecuda.Context(4096, PIR_MODULI, 17)
    c2 = hecuda.Context(8192, orc.generate_primes([55] * 4, False, 8192), 65537)
    benches = [KeyBench(name, ctx, pir.MulPir.generateParameter(config, ctx).evaluationKeyConfig.galoisElements)
               for name, ctx in (("n4096_27_28_28", pir_ctx), ("n8192_4x55", c2))]
    for kb in benches:
        print(json.dumps(kb.time(args.reps)), flush=True)
    if not args.skip_pir:
        bench_clients(pir_ctx, args.entries, args.clients, max(3, args.reps // 4))
    for kb in benches:  # profiler passes last
        print(json.dumps(kb.kernels(args.reps)), flush=True)
    c2.close()
    pir_ctx.close()


if __name__ == "__main__":
    main()
