#!/usr/bin/env python
"""A few MulPir queries at the BASELINE config 4 shape (2^20 x 64 B, default 27/28/28-bit parameters), for an ncu capture of
the first-dimension scan:  ncu --set full -k regex:inner_product_plain python tools/prof_pir_scan.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "swift-homomorphic-encryption_b200")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import hecuda
from hecuda import pir
from bench_pir import PIR_MODULI, uniform

n, t = 4096, 17
ctx = hecuda.Context(n, PIR_MODULI, t)
L = ctx.L
rng = np.random.default_rng(3)
config = pir.IndexPirConfig(1 << 20, 64, 2, 1, True, "hybridCompression", False)
param = pir.MulPir.generateParameter(config, ctx)
count = int(np.prod(param.dimensions))
db = pir.ProcessedDatabase(ctx, rng.integers(0, t, size=(count, n), dtype=np.uint64), None, evalFormat=False)
server = pir.MulPirServer(param, ctx, [db])
key = hecuda.EvaluationKey(ctx, uniform(rng, PIR_MODULI, (L, 2), n))
for e in param.evaluationKeyConfig.galoisElements:
    key.setGaloisKey(e, uniform(rng, PIR_MODULI, (L, 2), n))
query = uniform(rng, PIR_MODULI[:L], (-(-param.expandedQueryCount // n), 2), n)
for _ in range(4):
    server.computeResponse(query, key)
print("done", param.dimensions, count)
