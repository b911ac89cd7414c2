"""CPU check of the Montgomery reduction for primes h 2^32 + 1 (csrc/modarith.cuh: mont_reduce_h), which the lift,
floor and tensor kernels use modulo the multiply's 55-bit auxiliary primes.  It must return exactly what mont_reduce
returns, so the conditional subtractions after it see the same numbers: checked at the auxiliary primes of C2 and
C2-L4 over random accumulators, accumulators with a zero low word, and the largest sums each kernel forms."""
import os
import random
import shutil
import subprocess

import pytest

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "mont_reduce_h.cpp")
CXX = shutil.which("g++") or shutil.which("c++")
M64 = (1 << 64) - 1

# the largest 55-bit NTT primes for N = 8192 (bench.py's C2 uses the first four, C2-L4 the first five)
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417, 36028797017014273]


def aux_primes(moduli):
    """context.cu's 55-bit auxiliary base: the L + 1 smallest 55-bit primes h 2^32 + 1 that are not coefficient moduli."""
    L = len(moduli) - 1
    out, c = [], (1 << 54) + 1
    while len(out) < L + 1:
        if orc.is_prime(c) and c not in moduli:
            out.append(c)
        c += 1 << 32
    return out


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if CXX is None:
        pytest.skip("no C++ compiler")
    binary = str(tmp_path_factory.mktemp("mont") / "mont_reduce_h")
    subprocess.check_call([CXX, "-O2", "-std=c++17", "-o", binary, SRC])
    return binary


def exact(acc, p):
    """mont_reduce's definition: (acc + m p) / 2^64 with m = acc (-p^-1) mod 2^64, modulo 2^64."""
    m = (acc * (-pow(p, -1, 1 << 64))) & M64
    return ((acc + m * p) >> 64) & M64


def accumulators(p, qmax, L, rng):
    b = p
    accs = [
        (2**32 + b - 1) * (b - 1) + L * (qmax - 1) * (b - 1),  # lift: r_c qr[j] + sum_i z_i mat[j][i]
        2 * (b - 1) ** 2,                                      # tensor: c1 = a0 b1 + a1 b0
        (b - 1) ** 2,                                          # tensor: c0, c2
        (b - 1) ** 2 + L * (qmax - 1) * (b - 1),               # floor: f_j
        (2 * b - 1) * (b - 1) + L * (b - 1) ** 2,              # floor: alpha (f_msk < 2 m_sk)
        0, 1, M64, 1 << 64, (1 << 64) | 1, (1 << 96), (1 << 127) - 1, (1 << 128) - 1,
    ]
    for _ in range(2000):
        accs.append(rng.getrandbits(128))
    for _ in range(200):
        accs.append(rng.getrandbits(64) << 64)                 # lo = 0
        accs.append(rng.getrandbits(96) << 32)                 # lo0 = 0, lo1 != 0
        accs.append((rng.getrandbits(64) << 64) | rng.getrandbits(32))  # lo1 = 0
    return accs


@pytest.mark.parametrize("nmod", [4, 5])
def test_mont_reduce_h_equals_mont_reduce(checker, nmod):
    moduli = Q8192[:nmod]
    L = nmod - 1
    rng = random.Random(nmod)
    rows, want = [], []
    for p in aux_primes(moduli):
        assert p % (1 << 32) == 1 and p < 1 << 55 and (p - 1) % (2 * 8192) == 0
        for acc in accumulators(p, max(moduli[:L]), L, rng):
            rows.append(f"{p} {acc >> 64} {acc & M64}")
            want.append(exact(acc, p))
    out = subprocess.run([checker], input="\n".join(rows) + "\n", capture_output=True, text=True, check=True).stdout
    got = [tuple(int(v) for v in line.split()) for line in out.splitlines()]
    assert len(got) == len(want)
    for row, w, (generic, special) in zip(rows, want, got):
        assert generic == w, row
        assert special == w, row
