"""Saving and loading processed PNNS databases (pnns.ProcessedDatabase.save / load, the reference's
SerializedProcessedDatabase protobuf file).

Shape: C5 -- 100 000 x 512 seeded standard-normal float32 vectors, N = 8192, three 55-bit ciphertext moduli plus a
55-bit key-switching modulus, t = 65537, one plaintext modulus (--rows / --cols change it).

One JSON line per measurement group; every value of `reps` runs after one warm-up run (milliseconds, host clock around
calls that end in a device synchronise):
  - load_pinned_ms / load_pageable_ms / load_file_ms: ProcessedDatabase.load from a pinned buffer, a pageable one and a
    page-cached np.memmap file, with the contexts given;
  - save_pinned_ms / save_pageable_ms: the serialization into a pinned and a pageable buffer;
  - load_c_pinned_ms / save_c_pinned_ms: the same pinned load and save as bare C-ABI calls
    (hecuda_pnns_matrices_create_serialized, hecuda_pnns_database_serialize), without the Python layer's describe and
    entry walks or its conversions of the 100 000 entry identifiers;
  - copy_ceiling_ms: one plain host-to-device copy of the same bytes from pinned memory (torch);
  - process_ms: ProcessedDatabase.processOnDevice from the same vectors;
  - kernels: per kernel name, the device time of one pinned load and one pinned save from torch.profiler, in a separate
    pass;
  - parity: at a reduced shape, the saved bytes equal the restatement (tests/pnns_database_io_ref.py) of the resident
    words, and a load of them is word for word the saved matrix.
The first line names the card and its power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tests")]

import hecuda  # noqa: E402
from hecuda import pnns  # noqa: E402

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "error": str(e)}


def sync():
    import torch
    torch.cuda.synchronize()


def timed(fn, reps):
    fn()  # warm-up
    sync()
    out = []
    for _ in range(reps):
        start = time.perf_counter()
        result = fn()
        sync()
        out.append(round((time.perf_counter() - start) * 1e3, 2))
        if isinstance(result, pnns.ProcessedDatabase):
            result.close()
    return out


def copy_ceiling(nbytes, reps):
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    return timed(lambda: dst.copy_(src, non_blocking=True), reps)


def profile(fn, outdir, tag):
    import torch
    from torch.profiler import ProfilerActivity
    with torch.profiler.profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        sync()
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name if "Memcpy" in e.name else e.name.split("<")[0].split("(")[0]
            kernels[name] = kernels.get(name, 0.0) + e.device_time_total / 1e3
    if outdir:
        prof.export_chrome_trace(os.path.join(outdir, f"pnns_database_io_{tag}.pt.trace.json"))
    return {k: round(v, 3) for k, v in sorted(kernels.items())}


def c_load(ctx, data):
    handles = (C.c_void_p * 1)()
    ctxs = (C.c_void_p * 1)(ctx._h.value)
    hecuda._check(hecuda.load_library().hecuda_pnns_matrices_create_serialized(
        ctxs, 1, data.ctypes.data_as(C.c_void_p), data.size, handles))
    hecuda.load_library().hecuda_pnns_matrix_destroy(handles[0])


def c_save(processed, out):
    args, keep = processed._entries()
    written = C.c_uint64(0)
    lib = hecuda.load_library()

    def run():
        assert keep is not None  # the buffers `args` points into live as long as this closure
        hecuda._check(lib.hecuda_pnns_database_serialize(*args, out.ctypes.data_as(C.c_void_p), out.size, C.byref(written)))
    return run


def setup(rows, cols, seed=5):
    ctx = hecuda.Context(8192, Q8192, 65537)
    params = pnns.EncryptionParameters(8192, 65537, tuple(Q8192))
    dims = pnns.MatrixDimensions(rows, cols)
    ekc = pnns.MatrixMultiplication.evaluationKeyConfig(dims, 1, 8192)
    cc = pnns.ClientConfig(params, pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, cols, [65537]), cols, ekc)
    sc = pnns.ServerConfig(cc)
    vectors = np.random.default_rng(seed).standard_normal((rows, cols)).astype(np.float32)
    db = pnns.Database([pnns.DatabaseRow(i, b"", v) for i, v in enumerate(vectors)])  # rows as float32 arrays
    return ctx, sc, db


def parity():
    from oracle import pir_oracle as opir  # noqa: F401  (the restatement's codec)
    import pnns_database_io_ref as ref
    from test_gpu_evk_wire import read_device
    ctx, sc, db = setup(700, 64, seed=9)
    processed = pnns.ProcessedDatabase.processOnDevice(db, sc, [ctx])
    m = processed.plaintextMatrices[0]
    words = read_device(*m.deviceBuffer())
    b = sc.babyStepGiantStep
    polys = ref.polys_from_resident(8192, Q8192[:3], words, 700, 64, (b.vectorDimension, b.babyStep, b.giantStep))
    cfg = {"client_config": {
        "encryption_parameters": {"polynomial_degree": 8192, "plaintext_modulus": 65537, "coefficient_moduli": Q8192,
                                  "he_scheme": 1},
        "scaling_factor": sc.scalingFactor, "query_packing": ("denseRow",), "vector_dimension": 64,
        "galois_elements": list(sc.evaluationKeyConfig.galoisElements), "extra_plaintext_moduli": []},
        "database_packing": ("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))}
    matrices = [{"num_rows": 700, "num_columns": 64, "plaintexts": polys,
                 "packing": ("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))}]
    expected = ref.encode_processed_database(matrices, processed.entryIds, processed.entryMetadatas, cfg)
    data = processed.serialize()
    loaded = pnns.ProcessedDatabase.load(data, [ctx])
    same = bool(np.array_equal(read_device(*loaded.plaintextMatrices[0].deviceBuffer()), words))
    loaded.close(), processed.close()
    return {"bytes": len(data), "save_equals_restatement": data == expected, "load_equals_saved": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100000)
    ap.add_argument("--cols", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    a = ap.parse_args()
    print(json.dumps(card()), flush=True)
    print(json.dumps({"parity": parity()}), flush=True)
    ctx, sc, db = setup(a.rows, a.cols)
    process_ms = timed(lambda: pnns.ProcessedDatabase.processOnDevice(db, sc, [ctx]), a.reps)
    processed = pnns.ProcessedDatabase.processOnDevice(db, sc, [ctx])
    size = processed.serializationByteCount()
    resident_bytes = processed.plaintextMatrices[0].deviceBuffer()[1]
    pinned = hecuda.PinnedBuffer((size,), np.uint8)
    pageable = np.empty(size, dtype=np.uint8)
    processed._serialize_into(pinned.array)
    pageable[:] = pinned.array
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "c5.binpb")
        processed.save(path)
        result = {
            "shape": {"rows": a.rows, "cols": a.cols, "file_bytes": size, "resident_bytes": resident_bytes},
            "load_pinned_ms": timed(lambda: pnns.ProcessedDatabase.load(pinned.array, [ctx]), a.reps),
            "load_pageable_ms": timed(lambda: pnns.ProcessedDatabase.load(pageable, [ctx]), a.reps),
            "load_file_ms": timed(lambda: pnns.ProcessedDatabase.load(path, [ctx]), a.reps),
            "save_pinned_ms": timed(lambda: processed._serialize_into(pinned.array), a.reps),
            "load_c_pinned_ms": timed(lambda: c_load(ctx, pinned.array), a.reps),
            "save_c_pinned_ms": timed(c_save(processed, pinned.array), a.reps),
            "save_pageable_ms": timed(lambda: processed._serialize_into(pageable), a.reps),
            "copy_ceiling_ms": copy_ceiling(size, a.reps),
            "process_ms": process_ms,
        }
    print(json.dumps(result), flush=True)
    kernels = {"load": profile(lambda: pnns.ProcessedDatabase.load(pinned.array, [ctx]).close(), a.out, "load"),
               "save": profile(lambda: processed._serialize_into(pinned.array), a.out, "save")}
    print(json.dumps({"kernels": kernels}), flush=True)
    pinned.free()
    processed.close()


if __name__ == "__main__":
    main()
