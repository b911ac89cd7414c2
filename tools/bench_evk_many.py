#!/usr/bin/env python
"""Many clients' seeded evaluation keys in one call (hecuda_evk_create_serialized_many) against one
hecuda_evk_create_serialized call per client.

    python tools/bench_evk_many.py [--reps R] [--counts 1,4,16,64,256]

At the two key shapes of DESIGN.md section 6 (N = 4096, q = 27/28/28 bits with the 5 Galois elements of the PIR
default parameters; N = 8192, 4 x 55 bits with 2), for every K: keys/s of one _many call and of K single calls,
alternated in the same run, each from pinned and from pageable client buffers (host calls, the final synchronise
included, the destruction of the keys excluded); a plain pinned host-to-device copy of the same K keys' wire bytes as
the ceiling; kernel launches per call; device memory per key; the cudaMalloc of one key's device allocation; and, in a
separate torch.profiler pass, the device time of the DRBG chain and expansion kernels per _many call.  Every client has
its own buffers (copies of a few generated keys).  Prints one JSON line per measurement, and the card's name and
power limit read in the same run.  Key values are uniform residues: the load does not depend on them being
well-formed."""
import argparse
import ctypes as C
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
KEY_KERNELS = ("drbg_chain_kernel", "key_expand_kernel")
POOL = 8  # distinct generated keys; client j's buffers are copies of key j % POOL


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def wire_bytes(ctx, rng, cts):
    """One client's key ciphertexts on the wire: poly0 (cts x B) and seeds (cts x 32), from uniform residues."""
    words = np.empty((cts, ctx.L + 1, ctx.degree), dtype=np.uint64)
    for i, q in enumerate(ctx.coefficientModuli):
        words[:, i, :] = rng.integers(0, q, size=(cts, ctx.degree), dtype=np.uint64)
    poly0 = hecuda.Bfv.serialize(ctx, words, base=hecuda.BASE_KEYSWITCH)
    return np.ascontiguousarray(poly0.reshape(-1)), rng.integers(0, 256, size=cts * 32, dtype=np.uint8)


class Clients:
    """K clients' wire keys in their own buffers, pinned (hecuda_host_alloc) or pageable."""

    def __init__(self, pool, k, pinned):
        self.pins = []
        self.poly0, self.seeds = [], []
        for j in range(k):
            p, s = pool[j % len(pool)]
            if pinned:
                b = hecuda.PinnedBuffer(p.shape, np.uint8)
                b.array[:] = p
                self.pins.append(b)
                p = b.array
            else:
                p = p.copy()
            self.poly0.append(p)
            self.seeds.append(s.copy())
        self.poly0_ptrs = (C.c_void_p * k)(*[a.ctypes.data for a in self.poly0])
        self.seeds_ptrs = (C.c_void_p * k)(*[a.ctypes.data for a in self.seeds])

    def close(self):
        self.poly0 = None
        for b in self.pins:
            b.free()


class Shape:
    def __init__(self, name, ctx, elements):
        self.name, self.ctx, self.elements = name, ctx, np.ascontiguousarray(elements, dtype=np.uint32)
        L, n = ctx.L, ctx.degree
        self.cts = (1 + len(elements)) * L
        self.B = hecuda.Bfv.serializationByteCount(ctx, L + 1, base=hecuda.BASE_KEYSWITCH)
        rng = np.random.default_rng(7)
        self.pool = [wire_bytes(ctx, rng, self.cts) for _ in range(POOL)]
        self.wire_bytes = self.cts * (self.B + 32)
        self.key_device_bytes = (1 + len(elements)) * L * 2 * (L + 1) * n * 8
        self.lib = hecuda.load_library()

    def many(self, cl, k):
        out = (C.c_void_p * k)()
        rc = self.lib.hecuda_evk_create_serialized_many(self.ctx._h, k, 1, self.elements.ctypes.data, len(self.elements),
                                                        cl.poly0_ptrs, cl.seeds_ptrs, out)
        assert rc == 0, self.lib.hecuda_last_error()
        return list(out)

    def singles(self, cl, k):
        out, L = [], self.ctx.L
        for j in range(k):
            h = C.c_void_p()
            p, s = cl.poly0[j].ctypes.data, cl.seeds[j].ctypes.data
            rc = self.lib.hecuda_evk_create_serialized(self.ctx._h, p, s, self.elements.ctypes.data, len(self.elements),
                                                       p + L * self.B, s + L * 32, C.byref(h))
            assert rc == 0, self.lib.hecuda_last_error()
            out.append(h.value)
        return out

    def destroy(self, handles):
        for h in handles:
            self.lib.hecuda_evk_destroy(C.c_void_p(h))


def timed(shape, fn, cl, k):
    t0 = time.perf_counter()
    handles = fn(cl, k)
    dt = time.perf_counter() - t0
    shape.destroy(handles)
    return dt


def bench_count(shape, k, reps):
    """One _many call against k single calls, alternated, from pinned and pageable client buffers."""
    sources = {"pinned": Clients(shape.pool, k, True), "pageable": Clients(shape.pool, k, False)}
    times = {(m, s): [] for m in ("many", "single") for s in sources}
    launches = {}
    for r in range(reps + 1):  # the first round warms up
        for m, fn in (("many", shape.many), ("single", shape.singles)):
            for s, cl in sources.items():
                before = hecuda.kernel_launch_count()
                dt = timed(shape, fn, cl, k)
                launches[m] = (hecuda.kernel_launch_count() - before) / (1 if m == "many" else k)
                if r:
                    times[(m, s)].append(dt)
    # the ceiling: one pinned host-to-device copy of the same wire bytes
    host = torch.empty(k * shape.wire_bytes, dtype=torch.uint8).pin_memory()
    dev = torch.empty_like(host, device="cuda")
    dev.copy_(host, non_blocking=True)
    torch.cuda.synchronize()
    copy = []
    for _ in range(reps):
        t0 = time.perf_counter()
        dev.copy_(host, non_blocking=True)
        torch.cuda.synchronize()
        copy.append(time.perf_counter() - t0)
    for cl in sources.values():
        cl.close()
    med = {key: float(np.median(v)) for key, v in times.items()}
    return dict(measure="evk_many", shape=shape.name, keys=k, elements=len(shape.elements), key_ciphertexts=shape.cts,
                wire_bytes_per_key=shape.wire_bytes, device_bytes_per_key=shape.key_device_bytes,
                launches_per_many_call=launches["many"], launches_per_single_call=launches["single"],
                keys_per_s={f"{m}_{s}": k / med[(m, s)] for (m, s) in med},
                pinned_copy_keys_per_s=k / float(np.median(copy)),
                pinned_copy_gb_per_s=k * shape.wire_bytes / float(np.median(copy)) / 1e9)


def bench_alloc(shape, reps):
    """cudaMalloc + cudaFree of one key's device allocation, through the runtime the library uses."""
    rt = C.CDLL("libcudart.so.12")
    p = C.c_void_p()
    allocs, frees = [], []
    for r in range(reps + 1):
        t0 = time.perf_counter()
        assert rt.cudaMalloc(C.byref(p), C.c_size_t(shape.key_device_bytes)) == 0
        t1 = time.perf_counter()
        assert rt.cudaFree(p) == 0
        t2 = time.perf_counter()
        if r:
            allocs.append(t1 - t0)
            frees.append(t2 - t1)
    return dict(measure="evk_alloc", shape=shape.name, device_bytes_per_key=shape.key_device_bytes,
                cudaMalloc_us=float(np.median(allocs)) * 1e6, cudaFree_us=float(np.median(frees)) * 1e6)


def bench_kernels(shape, k, reps):
    """Device time of the chain and expansion kernels per _many call of k keys.  Run after every timing: the profiler
    slows later runtime calls."""
    cl = Clients(shape.pool, k, True)
    shape.destroy(shape.many(cl, k))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            shape.destroy(shape.many(cl, k))
        torch.cuda.synchronize()
    cl.close()
    us = {name: 0.0 for name in KEY_KERNELS}
    for ev in prof.key_averages():
        for name in KEY_KERNELS:
            if name in ev.key:
                us[name] += ev.device_time_total / reps
    return dict(measure="evk_many_kernels", shape=shape.name, keys=k, kernels_us_per_call=us,
                expand_us_per_key=us["key_expand_kernel"] / k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--counts", default="1,4,16,64,256")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evk_many needs a CUDA device")
    counts = [int(x) for x in args.counts.split(",")]
    print(json.dumps(dict(card=card())), flush=True)
    from oracle import oracle as orc

    config = pir.IndexPirConfig(1 << 20, 64, 2, 1, True, "hybridCompression", False)
    pir_ctx = hecuda.Context(4096, PIR_MODULI, 17)
    c2 = hecuda.Context(8192, orc.generate_primes([55] * 4, False, 8192), 65537)
    shapes = [Shape("n4096_27_28_28", pir_ctx, pir.MulPir.generateParameter(config, pir_ctx).evaluationKeyConfig.galoisElements),
              Shape("n8192_4x55", c2, pir.MulPir.generateParameter(config, c2).evaluationKeyConfig.galoisElements)]
    for sh in shapes:
        print(json.dumps(bench_alloc(sh, 20)), flush=True)
        for k in counts:
            print(json.dumps(bench_count(sh, k, args.reps)), flush=True)
    for sh in shapes:  # profiler passes last
        for k in (counts[0], counts[-1]):
            print(json.dumps(bench_kernels(sh, k, 3)), flush=True)
    c2.close()
    pir_ctx.close()


if __name__ == "__main__":
    main()
