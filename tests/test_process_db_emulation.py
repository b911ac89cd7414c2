"""CPU-side verification of the database-processing kernels' index maps (csrc/process_db.cuh).

tests/emu/process_db_emulate.cu evaluates the very same __host__ __device__ functions that the MulPir packing kernel and
the PNNS diagonal-gather kernel call, and the results must equal the host ports:
  - MulPirServer.plaintextRows (rows and presence flags), for the pack and split paths;
  - PlaintextMatrix.diagonalPlaintexts' SIMD slot values (decoded back from its plaintexts), in diagonalPlaintexts' order
    and in hecuda_pnns_matrix_create's resident slot order."""
import os
import random
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from hecuda import pir, pnns

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "process_db_emulate.cu")
HDR = os.path.join(ROOT, "swift-homomorphic-encryption_b200", "csrc", "process_db.cuh")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "process_db_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, args, text):
    return subprocess.run([binary] + [str(a) for a in args], input=text, capture_output=True, text=True,
                          check=True).stdout.splitlines()


def emulate_pir(binary, ctx, param, database, offsets):
    dims = param.dimensions
    args = ["pir", ctx.degree, ctx.plaintextModulus, param.entrySizeInBytes, int(param.encodingEntrySize), len(dims), *dims,
            len(database), int(offsets)]
    lines = run(binary, args, "".join((bytes(e).hex() or ".") + "\n" for e in database))
    table = np.array([[int(v) for v in line.split()] for line in lines], dtype=np.uint64)
    return table[:, 1:], table[:, 0].astype(np.uint8)


# (N, t, entry size, entry count, dimensions, encodingEntrySize, variable-length entries)
PIR_CASES = [
    (16, 17, 1, 40, 1, False, False),
    (16, 17, 1, 40, 2, True, True),
    (16, 2 ** 23 + 16385, 5, 30, 1, True, False),
    (16, 1153, 47, 30, 2, True, True),          # 3 chunks per entry
    (64, 1153, 8, 100, 2, False, False),
    (64, 1153, 24, 50, 1, True, True),
    (64, 17, 3000, 4, 1, False, False),         # 94 chunks per entry
    (64, 786433, 7, 61, 2, False, False),
    (256, 65537, 100, 70, 2, False, False),
    (256, 40961, 255, 21, 2, True, True),       # 255 bytes still take a 1-byte prefix
    (256, 40961, 256, 21, 1, True, True),       # 256 bytes take a 2-byte prefix
    (1024, 2 ** 23 + 16385, 3000, 9, 2, True, True),
    (4096, 17, 64, 300, 2, False, False),
]


@pytest.mark.parametrize("n,t,size,entries,dims,encoding,variable", PIR_CASES)
def test_pir_packing_matches_plaintext_rows(emu, n, t, size, entries, dims, encoding, variable):
    ctx = SimpleNamespace(degree=n, plaintextModulus=t)
    param = pir.MulPir.generateParameter(
        pir.IndexPirConfig(entries, size, dims, 1, False, "noCompression", encoding), ctx)
    rng = random.Random(n * 7919 + size)
    database = []
    for i in range(entries):
        length = rng.randint(0, size) if variable else size
        if i % 7 == 3:
            database.append(bytes(length))          # all-zero entries
        else:
            database.append(bytes(rng.randrange(256) for _ in range(length)))
    if variable:
        database[0] = b""
        database[-1] = bytes(rng.randrange(256) for _ in range(size))
    rows, present = pir.MulPirServer.plaintextRows(database, ctx, param)
    for offsets in ((True, False) if not variable else (True,)):
        got_rows, got_present = emulate_pir(emu, ctx, param, database, offsets)
        assert got_rows.shape == rows.shape
        assert np.array_equal(got_rows, rows)
        assert np.array_equal(got_present, present)


def pnns_slots(binary, n, rows, cols, bsgs, t, values, reduce, resident):
    args = ["pnns", n.bit_length() - 1, rows, cols, bsgs.babyStep, bsgs.giantStep, t, int(reduce), int(resident)]
    lines = run(binary, args, " ".join(str(int(v)) for v in np.asarray(values).reshape(-1)) + "\n")
    bad = lines[0] == "bad 1"
    return bad, np.array([[int(v) for v in line.split()] for line in lines[1:]], dtype=np.uint64)


# (N, t, rows, cols, (babyStep, giantStep) or None for forVectorDimension)
PNNS_CASES = [
    (16, 97, 5, 3, None),
    (16, 97, 16, 5, None),
    (16, 97, 37, 7, (8, 1)),
    (16, 97, 37, 7, (3, 3)),
    (16, 97, 40, 8, (4, 2)),
    (64, 65537, 63, 20, None),
    (64, 65537, 64, 32, (8, 4)),
    (64, 65537, 150, 17, (32, 1)),
    (4096, 65537, 5000, 3, None),
]


@pytest.mark.parametrize("n,t,rows,cols,steps", PNNS_CASES)
@pytest.mark.parametrize("reduce", [False, True])
def test_pnns_gather_matches_diagonal_plaintexts(emu, n, t, rows, cols, steps, reduce):
    dimension = pnns._next_power_of_two(cols)
    bsgs = pnns.BabyStepGiantStep(dimension, *steps) if steps else pnns.BabyStepGiantStep.forVectorDimension(cols)
    rng = np.random.default_rng(rows * 131 + cols)
    if reduce:
        values = rng.integers(-(1 << 40), 1 << 40, size=(rows, cols), dtype=np.int64)
        values[0, 0], values[-1, -1] = np.iinfo(np.int64).min, np.iinfo(np.int64).max
        remainders = np.array([int(v) % t for v in values.reshape(-1)], dtype=np.uint64)
    else:
        values = rng.integers(-(t // 2), (t - 1) // 2 + 1, size=(rows, cols), dtype=np.int64)
        values[0, 0], values[-1, -1] = -(t // 2), (t - 1) // 2
        remainders = pnns.centeredToRemainder(values, t).reshape(-1)
    ctx = SimpleNamespace(degree=n, plaintextModulus=t)
    dims = pnns.MatrixDimensions(rows, cols)
    plaintexts = pnns.PlaintextMatrix.diagonalPlaintexts(ctx, dims, bsgs, remainders)
    expected = pnns.SimdEncoder(n, t).decode(plaintexts)
    bad, slots = pnns_slots(emu, n, rows, cols, bsgs, t, values, reduce, False)
    assert not bad
    assert np.array_equal(slots, expected)
    # resident order: plaintext results * (j + babyStep * g) + r  ->  slot (r * giantStep + g) * babyStep + j
    bad, resident = pnns_slots(emu, n, rows, cols, bsgs, t, values, reduce, True)
    results = -(-rows // n)
    assert not bad and resident.shape[0] == results * bsgs.giantStep * bsgs.babyStep
    for r in range(results):
        for g in range(bsgs.giantStep):
            for j in range(bsgs.babyStep):
                slot = (r * bsgs.giantStep + g) * bsgs.babyStep + j
                d = bsgs.babyStep * g + j
                want = expected[results * d + r] if d < dimension else np.zeros(n, dtype=np.uint64)
                assert np.array_equal(resident[slot], want), (r, g, j)


@pytest.mark.parametrize("value", [-49, 49, 1 << 62, -(1 << 62)])
def test_pnns_out_of_range_values_are_flagged(emu, value):
    t = 97  # centered range [-48, 48]
    values = np.zeros((5, 3), dtype=np.int64)
    values[2, 1] = value
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(3)
    assert pnns_slots(emu, 16, 5, 3, bsgs, t, values, False, False)[0]
    assert not pnns_slots(emu, 16, 5, 3, bsgs, t, values, True, False)[0]
    values[2, 1] = 48
    assert not pnns_slots(emu, 16, 5, 3, bsgs, t, values, False, False)[0]
