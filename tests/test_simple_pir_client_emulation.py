"""CPU replay of the SimplePIR client's helpers (csrc/simple_pir.cuh, process_db.cuh) through
tests/emu/simple_pir_client_emulate.cu, against Python integers:

- the stream coefficients of secret (i, j) and error (i, c);
- add(index:)'s column and extractEntries' gather, for chunksPerEntry 1 and entriesPerColumn 1;
- divideAndRound(p -> 2^ct) at x = 0, p - 1, at rounding ties and at random x;
- the results epilogue with every plane sum at N x 255 under both masks, for 32- and 64-bit scalars, where the double-
  width sum wraps;
- integrate and coefficientsToBytes at pt = 1 .. ct - 1."""
import os
import random
import shutil
import subprocess

import pytest

from oracle import simple_pir_oracle as osp
from oracle.pir_oracle import coefficients_to_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "simple_pir_client_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "simple_pir_client_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, lines):
    out = subprocess.run([binary], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    return out.split("\n")[:len(lines)]


def test_stream_offsets(emu):
    cases = [(i, j, n, c, k) for i in range(3) for n in (8, 2048) for j in (0, n - 1) for k in (7, 1 << 20) for c in (0, k - 1)]
    got = run(emu, [f"offsets {i} {j} {n} {c} {k}" for i, j, n, c, k in cases])
    assert got == [f"{i * n + j} {i * k + c}" for i, j, n, c, k in cases]


def test_delta_column_and_extract_gather(emu):
    cases = []
    for cpe, epc in ((1, 1), (1, 5), (3, 1), (6, 1)):
        for index in (0, 1, 7, 1000):
            for i in range(cpe):
                cases.append((index, i, cpe, epc))
    got = run(emu, [f"delta {ix} {i} {cpe} {epc}" for ix, i, cpe, epc in cases])
    assert got == [str((ix * cpe + i) // epc) for ix, i, cpe, epc in cases]
    lines, expect = [], []
    for index, i, cpe, epc in cases:
        chunk = 11
        m = epc * chunk
        for t in (0, chunk - 1):
            lines.append(f"extract {index} {i} {t} {cpe} {epc} {m} {chunk}")
            expect.append(str(i * m + ((index * cpe + i) % epc) * chunk + t))  # extractEntries' indexStart + t
    assert run(emu, lines) == expect


@pytest.mark.parametrize("ct,n", [(9, 8), (28, 1024), (31, 1024), (42, 2048), (61, 2048)])
def test_divide_and_round(emu, ct, n):
    p = osp.ntt_friendly_mod(ct, n)
    xs = [0, 1, p - 1, p // 2, p // 2 + 1]
    # ties: x 2^ct + floor(p / 2) = q p exactly lands on a quotient boundary
    for q in (1, 2, (1 << ct) - 1):
        xs += [x for x in ((q * p - p // 2) >> ct, ((q * p - p // 2) >> ct) + 1) if 0 <= x < p]
    rng = random.Random(ct)
    xs += [rng.randrange(p) for _ in range(50)]
    got = run(emu, [f"round {x} {p} {ct}" for x in xs])
    assert got == [str(((x << ct) + (p >> 1)) // p % (1 << ct)) for x in xs]


@pytest.mark.parametrize("w,ct,n", [(32, 28, 1024), (32, 31, 1024), (64, 42, 2048), (64, 61, 2048), (64, 61, 1 << 15)])
def test_results_epilogue_wraps_like_the_reference(emu, w, ct, n):
    p = osp.ntt_friendly_mod(ct, min(n, 2048))
    planes = (ct + 1 + 7) // 8
    rng = random.Random(w + ct)
    cases = [[(n * 255, n * 255)] * planes, [(n * 255, 0)] * planes, [(0, n * 255)] * planes]
    cases += [[(rng.randrange(n * 255 + 1), rng.randrange(n * 255 + 1)) for _ in range(planes)] for _ in range(20)]
    lines, expect, wrapped = [], [], 0
    for sums in cases:
        lines.append(f"results {w} {p} {planes} " + " ".join(f"{a} {b}" for a, b in sums))
        u = sum((a + (p - 1) * b) << (8 * d) for d, (a, b) in enumerate(sums))
        wrapped += u >= 1 << (2 * w)
        expect.append(str(u % (1 << (2 * w)) % p))
    assert run(emu, lines) == expect
    largest = sum((n * 255 * p) << (8 * d) for d in range(planes))  # every sum at N x 255 under both masks
    assert (wrapped > 0) == (largest >= 1 << (2 * w))


@pytest.mark.parametrize("ct", [9, 28, 42, 61])
def test_integrate_and_coefficients_to_bytes(emu, ct):
    rng = random.Random(ct)
    lines, expect = [], []
    for pt in range(1, ct):
        delta, mask = 1 << (ct - pt), (1 << ct) - 1
        for r, s in ((0, 0), (mask, 0), (0, mask), (delta // 2, 0), (rng.randrange(1 << ct), rng.randrange(1 << ct))):
            lines.append(f"integrate {r} {s} {pt} {ct}")
            expect.append(str(((r - s + (delta >> 1)) & mask) >> (ct - pt)))
        count = rng.randrange(1, 20)
        coeffs = [rng.randrange(1 << pt) for _ in range(count)]
        lines.append(f"bytes {pt} {count} " + " ".join(map(str, coeffs)))
        expect.append(coefficients_to_bytes(coeffs, pt).hex())
    assert run(emu, lines) == expect
