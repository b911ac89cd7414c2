"""Saving and loading processed PIR databases (ProcessedDatabase.save / load, ProcessedKeywordDatabase.save / load).

Shapes (synthetic, seeded):
  c4       MulPir 2^20 x 64 B at the C4 context (N = 4096, t = 17, 27/28/28-bit moduli, the last one the key-switching
           modulus, uneven 2 dimensions): uint32 rows
  n8192    an index database of --n8192-plaintexts random Eval plaintexts at N = 8192 over 4 x 55-bit ciphertext moduli
           (and a 55-bit key-switching modulus), 225 280 B per plaintext: uint64 rows
  keyword  2^20 x 64 B keyword rows at the C4 context (defaultKeywordPir cuckoo table, 2 dimensions)

Per shape one JSON line, every value of `reps` runs after one warm-up run (milliseconds, host clock around calls that end
in a device synchronise):
  - load_pinned_ms / load_pageable_ms / load_file_ms: ProcessedDatabase.load from a pinned buffer, a pageable one and
    a page-cached np.memmap file;
  - save_pinned_ms / save_pageable_ms: the serialization into a pinned and a pageable buffer;
  - copy_ceiling_ms: one plain host-to-device copy of the same bytes from pinned memory (torch), the bound a load is
    judged against;
  - composed_ms (c4, n8192): the composed Python path the C ABI replaces -- host tag walk, hecuda_poly_load to uint64
    words on the host, then hecuda_pir_database_create(eval_format = 1);
  - process_ms (keyword): KeywordPirServer.processOnDevice, against load;
  - kernels: per kernel name, the device time of one pinned load and one pinned save from torch.profiler, in a
    separate pass;
  - parity: the saved bytes equal the reference serialization (tests/pir_database_io_ref.py) at a reduced shape.
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
from hecuda import keyword_pir as kw  # noqa: E402
from hecuda import pir  # noqa: E402

PIR_MODULI = [134176769, 268369921, 268361729]
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
        if isinstance(result, list):  # loaded databases
            for db in result:
                db.close()
    return out


def serialize_into(dbs, out):
    handles = (C.c_void_p * len(dbs))(*[d._h for d in dbs])
    written = C.c_uint64(0)
    hecuda._check(hecuda.load_library().hecuda_pir_databases_serialize(handles, len(dbs), out.ctypes.data_as(C.c_void_p),
                                                                        out.size, C.byref(written)))


def copy_ceiling(nbytes, reps):
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    return timed(lambda: dst.copy_(src, non_blocking=True), reps)


def composed_load(g, data):
    """What a caller had to compose before: the tag walk on the host, hecuda_poly_load of the present plaintexts to
    uint64 words, and hecuda_pir_database_create of the full count x L x N rows."""
    lib = hecuda.load_library()
    size = C.c_uint64(0)
    hecuda._check(lib.hecuda_poly_serialized_byte_count(g._h, hecuda.BASE_Q, g.L, 0, C.byref(size)))
    size = size.value
    count = int.from_bytes(data[1:5].tobytes(), "little")
    present = np.zeros(count, dtype=np.uint8)
    starts, at = [], 5
    for i in range(count):
        if data[at]:
            present[i] = 1
            starts.append(at + 1)
            at += 1 + size
        else:
            at += 1
    packed = np.empty((len(starts), size), dtype=np.uint8)
    for k, start in enumerate(starts):
        packed[k] = data[start:start + size]
    words = np.empty((len(starts), g.L, g.degree), dtype=np.uint64)
    hecuda._check(lib.hecuda_poly_load(g._h, hecuda.BASE_Q, hecuda._ptr(packed), 0, hecuda._ptr(words), g.L, len(starts)))
    rows = np.zeros((count, g.L, g.degree), dtype=np.uint64)
    rows[present == 1] = words
    return [pir.ProcessedDatabase(g, rows, present, evalFormat=True)]


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
        prof.export_chrome_trace(os.path.join(outdir, f"pir_database_io_{tag}.pt.trace.json"))
    return {k: round(v, 3) for k, v in sorted(kernels.items())}


def measure(name, g, dbs, table_count, reps, outdir, extra):
    data = pir._serialize_databases(dbs)
    pinned = hecuda.PinnedBuffer((data.size,), np.uint8)
    pinned.array[:] = data
    path = os.path.join(tempfile.mkdtemp(), f"{name}.bin")
    data.tofile(path)
    with open(path, "rb") as f:  # page cache
        while f.read(1 << 26):
            pass
    line = {"shape": name, "bytes": int(data.size), "plaintexts": sum(d.count for d in dbs),
            "resident_bytes": sum(d.deviceBuffer()[1] for d in dbs), **extra}
    line["load_pinned_ms"] = timed(lambda: pir.ProcessedDatabase.load(g, pinned.array, table_count), reps)
    line["load_pageable_ms"] = timed(lambda: pir.ProcessedDatabase.load(g, data, table_count), reps)
    line["load_file_ms"] = timed(lambda: pir.ProcessedDatabase.load(g, path, table_count), reps)
    line["save_pinned_ms"] = timed(lambda: serialize_into(dbs, pinned.array), reps)
    pageable = np.empty_like(data)
    line["save_pageable_ms"] = timed(lambda: serialize_into(dbs, pageable), reps)
    assert pageable.tobytes() == data.tobytes() and pinned.array.tobytes() == data.tobytes()
    line["copy_ceiling_ms"] = copy_ceiling(int(data.size), reps)
    if table_count == 1:
        line["composed_ms"] = timed(lambda: composed_load(g, data), max(1, reps // 2))
    loaded = pir.ProcessedDatabase.load(g, pinned.array, table_count)
    line["load_equal"] = all(np.array_equal(hecuda_words(a), hecuda_words(b)) and
                             np.array_equal(a.presentFlags(), b.presentFlags()) for a, b in zip(loaded, dbs))
    for d in loaded:
        d.close()
    line["kernels_load"] = profile(lambda: [d.close() for d in pir.ProcessedDatabase.load(g, pinned.array, table_count)],
                                   outdir, name + "_load")
    line["kernels_save"] = profile(lambda: serialize_into(dbs, pinned.array), outdir, name + "_save")
    pinned.free()
    os.remove(path)
    return line


def hecuda_words(db):
    import torch
    ptr, nbytes = db.deviceBuffer()

    class Buffer:
        __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}

    return torch.as_tensor(Buffer(), device="cuda").cpu().numpy()


def parity():
    """Saved bytes against the reference serialization at reduced shapes (a C4-context MulPir database and an N = 8192
    one)."""
    import pir_database_io_ref as ref
    out = {}
    for name, g, entries, size in (("c4_reduced", hecuda.Context(4096, PIR_MODULI, 17), 4096, 64),
                                   ("n8192_reduced", hecuda.Context(8192, Q8192, 65537), 300, 3000)):
        param = pir.MulPir.generateParameter(pir.IndexPirConfig(entries, size, 2, 1, True, "hybridCompression", False), g)
        rng = np.random.default_rng(entries)
        db = [bytes(r) for r in rng.integers(0, 256, size=(entries, size), dtype=np.uint8)]
        processed = pir.MulPirServer.processOnDevice(db, g, param)
        rows, present = pir.MulPirServer.plaintextRows(db, g, param)
        evals = hecuda.Bfv.plaintextToEval(g, rows)
        expected = ref.serialize_processed_database(g.degree, g.ciphertextModuli,
                                                    [evals[i] if present[i] else None for i in range(len(present))])
        out[name] = processed.serialize() == expected
        processed.close()
        g.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default="c4,n8192,keyword")
    ap.add_argument("--n8192-plaintexts", type=int, default=2000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if hecuda.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    print(json.dumps(card()), flush=True)
    shapes = args.shapes.split(",")
    if "c4" in shapes:
        g = hecuda.Context(4096, PIR_MODULI, 17)
        param = pir.MulPir.generateParameter(pir.IndexPirConfig(1 << 20, 64, 2, 1, True, "hybridCompression", False), g)
        raw = np.random.default_rng(20).integers(0, 256, size=(1 << 20, 64), dtype=np.uint8)
        db = pir.MulPirServer.processOnDevice([bytes(r) for r in raw], g, param)
        print(json.dumps(measure("c4", g, [db], 1, args.reps, args.out, {"dims": param.dimensions})), flush=True)
        db.close()
        g.close()
    if "n8192" in shapes:
        from oracle import oracle as orc
        g = hecuda.Context(8192, orc.generate_primes([55] * 5, False, 8192), 65537)
        count = args.n8192_plaintexts
        rng = np.random.default_rng(8192)
        rows = np.stack([rng.integers(0, q, size=(count, 8192), dtype=np.uint64) for q in g.ciphertextModuli], axis=1)
        db = pir.ProcessedDatabase(g, rows, np.ones(count, dtype=np.uint8), evalFormat=True)
        del rows
        print(json.dumps(measure("n8192", g, [db], 1, args.reps, args.out, {})), flush=True)
        db.close()
        g.close()
    if "keyword" in shapes:
        g = hecuda.Context(4096, PIR_MODULI, 17)
        rng = np.random.default_rng(64)
        keywords = rng.integers(0, 256, size=(1 << 20, 16), dtype=np.uint8)
        values = rng.integers(0, 256, size=(1 << 20, 64), dtype=np.uint8)
        rows = [(keywords[i].tobytes(), values[i].tobytes()) for i in range(1 << 20)]
        bpp = 4096 * 4 // 8
        single = kw.serializedSize(64)
        bucket = -(-single // bpp) * bpp if single >= bpp // 2 else bpp // 2
        config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(bucket), False, "hybridCompression")
        process_ms = []
        for rep in range(args.reps + 1):
            start = time.perf_counter()
            processed = kw.KeywordPirServer.processOnDevice(rows, config, g)
            sync()
            if rep:
                process_ms.append(round((time.perf_counter() - start) * 1e3, 2))
            if rep < args.reps:
                processed.close()
        extra = {"dims": processed.pirParameter.dimensions, "buckets": processed.table.bucketCount, "process_ms": process_ms}
        line = measure("keyword", g, processed.databases, config.parameter.hashFunctionCount, args.reps, args.out, extra)
        print(json.dumps(line), flush=True)
        processed.close()
        g.close()
    print(json.dumps({"parity": parity()}), flush=True)


if __name__ == "__main__":
    main()
