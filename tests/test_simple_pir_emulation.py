"""CPU replay of the SimplePIR response arithmetic (csrc/simple_pir.cuh) at its bounds.

tests/emu/simple_pir_emulate.cu runs the same __host__ __device__ digit split, slice widening and shift-and-mask
combine that response_kernel applies, and the results must equal (sum db * request) mod 2^ct in Python integers:
every DB digit 255, every request word 2^width - 1, a K-slice exactly full and one crossed, for
ct in {8, 9, 28, 31, 32, 33, 42, 61}.  The fragment layouts must be bijections onto their tiles."""
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "simple_pir_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
SLICE = 32768


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "simple_pir_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def emulate(binary, pt, ct, db, req):
    text = " ".join(map(str, db)) + "\n" + " ".join(map(str, req)) + "\n"
    out = subprocess.run([binary, "response", str(pt), str(ct), str(len(db))], input=text, capture_output=True, text=True, check=True)
    value, largest = out.stdout.split()
    return int(value), int(largest)


@pytest.mark.parametrize("ct", [8, 9, 28, 31, 32, 33, 42, 61])
@pytest.mark.parametrize("k", [SLICE, 2 * SLICE + 3])
def test_worst_case_operands(emu, ct, k):
    pt = min(16, ct - 1)
    width = 32 if ct < 32 else 64
    db = [(1 << pt) - 1] * k
    req = [(1 << width) - 1] * k
    value, largest = emulate(emu, pt, ct, db, req)
    assert value == sum(d * q for d, q in zip(db, req)) % (1 << ct)
    assert largest < (1 << 31)
    if pt >= 8:
        assert largest == 255 * 255 * SLICE  # the slice is exactly full at the bound


@pytest.mark.parametrize("pt,ct", [(7, 28), (8, 9), (9, 33), (14, 42), (16, 61)])
def test_random_operands(emu, pt, ct):
    rng = random.Random(pt * 100 + ct)
    k = SLICE + 77
    db = [rng.randrange(1 << pt) for _ in range(k)]
    req = [rng.randrange(1 << 64) for _ in range(k)]
    value, _ = emulate(emu, pt, ct, db, req)
    assert value == sum(d * q for d, q in zip(db, req)) % (1 << ct)


def test_fragment_layouts_are_bijections(emu):
    rows, cols = 32, 64
    out = subprocess.run([emu, "layout", str(rows), str(cols)], capture_output=True, text=True, check=True)
    offsets = [int(v) for v in out.stdout.split()]
    a, b = offsets[:rows * cols], offsets[rows * cols:]
    assert sorted(a) == list(range(rows * cols))
    assert sorted(b) == list(range(rows * cols))
    # a warp's A tile is one contiguous 512-byte block; row g of lane 4g + t holds columns 4t .. 4t + 3 at its start
    assert a[0 * cols + 0] == 0 and a[0 * cols + 4] == 16 and a[8 * cols + 0] == 4 and a[0 * cols + 16] == 8
    assert a[16 * cols + 0] == 2 * 512 and a[0 * cols + 32] == 512
    assert b[0 * cols + 4] == 8 and b[1 * cols + 0] == 32 and b[0 * cols + 16] == 4 and b[8 * cols + 0] == 2 * 256
