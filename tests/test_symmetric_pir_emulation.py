"""CPU-side verification of the symmetric-PIR device code (csrc/p384.cuh, csrc/sha512.cuh, csrc/aes_gcm.cuh).

tests/emu/symmetric_pir_emulate.cu evaluates the same __host__ __device__ functions the OPRF and seal kernels call, and
they are checked against oracle/oprf_oracle.py, hashlib and cryptography's AESGCM: field arithmetic at its edges, both
SSWU branches, scalars with long runs of equal windows, SHA-384 across its padding boundaries, OPRF inputs of length 0,
1 and 65535, and GCM values around the block size."""
import hashlib
import os
import random
import shutil
import subprocess

import pytest

from oracle import oprf_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "symmetric_pir_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "symmetric_pir_emulate")
    subprocess.check_call([NVCC, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, lines):
    out = subprocess.run([binary], input="".join(line + "\n" for line in lines), capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(lines)
    return out


def h48(x: int) -> str:
    return "%096x" % x


def hexb(b: bytes) -> str:
    return b.hex() or "."


def test_sha384_matches_hashlib(emu):
    rng = random.Random(5)
    messages = [rng.randbytes(n) for n in range(301)]
    for m, line in zip(messages, run(emu, ["sha384 " + hexb(m) for m in messages])):
        assert line == hashlib.sha384(m).hexdigest(), len(m)


def field_values():
    rng = random.Random(6)
    p = O.P
    edges = [0, 1, 2, p - 1, p - 2, 2**32 - 1, 2**32, 2**128, 2**383, p >> 1, (p + 1) // 2]
    carry = [sum(0xffffffff << (32 * i) for i in range(k)) % p for k in range(1, 13)]  # runs of all-ones limbs
    return edges + carry + [rng.randrange(p) for _ in range(30)]


def test_field_arithmetic(emu):
    p = O.P
    values = field_values()
    pairs = [(a, b) for a in values[:12] for b in values[:12]] + list(zip(values, reversed(values)))
    lines = []
    for a, b in pairs:
        lines += [f"mul {h48(a)} {h48(b)}", f"add {h48(a)} {h48(b)}", f"sub {h48(a)} {h48(b)}"]
    out = iter(run(emu, lines))
    for a, b in pairs:
        assert int(next(out), 16) == a * b % p
        assert int(next(out), 16) == (a + b) % p
        assert int(next(out), 16) == (a - b) % p
    nonzero = [v for v in values if v]
    for v, line in zip(nonzero, run(emu, [f"inv {h48(v)}" for v in nonzero])):
        assert int(line, 16) == pow(v, p - 2, p)


def test_sqrt_ratio_and_reduction(emu):
    rng = random.Random(7)
    cases = [(rng.randrange(O.P), rng.randrange(1, O.P)) for _ in range(30)] + [(0, 1), (1, 1), (O.P - 12, 1)]
    for (u, v), line in zip(cases, run(emu, [f"sqrt_ratio {h48(u)} {h48(v)}" for u, v in cases])):
        qr, y = line.split()
        assert (qr == "1", int(y, 16)) == O.sqrt_ratio(u, v)
    blobs = [bytes(72), b"\xff" * 72, O.P.to_bytes(72, "big"), (2 * O.P).to_bytes(72, "big")] + \
        [rng.randbytes(72) for _ in range(20)]
    for b, line in zip(blobs, run(emu, ["reduce72 " + b.hex() for b in blobs])):
        assert int(line, 16) == int.from_bytes(b, "big") % O.P


def test_sswu_both_branches(emu):
    rng = random.Random(8)
    us = [0, 1, O.P - 1] + [rng.randrange(O.P) for _ in range(40)]
    branches = set()
    for u, line in zip(us, run(emu, [f"map {h48(u)}" for u in us])):
        x, y, square = O.map_to_curve_sswu_generic(u)
        assert line.split() == [h48(x), h48(y), str(int(square))]
        branches.add(square)
    assert branches == {True, False}


def test_hash_to_group(emu):
    rng = random.Random(9)
    msgs = [b"", b"a", rng.randbytes(127), rng.randbytes(128), rng.randbytes(300)]
    for m, line in zip(msgs, run(emu, ["h2g " + hexb(m) for m in msgs])):
        x, y = O.hash_to_group(m)
        assert line.split() == [h48(x), h48(y)]


def scalars():
    rng = random.Random(10)
    n = O.N
    long_runs = [2**384 - 1 - 2**200, 2**383 + 1, (2**192 - 1) << 100 | 1, 0x10000000000000001, 16**95 + 1]
    return [1, 2, 3, 5, 6, n - 1, n - 2, n - 6, n - 7] + [k % n for k in long_runs] + [rng.randrange(1, n) for _ in range(8)]


def test_recoding(emu):
    ks = scalars()
    for k, line in zip(ks, run(emu, [f"recode {h48(k)}" for k in ks])):
        digits = [int(d) for d in line.split()]
        odd, flip = (k, 0) if k & 1 else (O.N - k, 1)
        assert digits == O.recode(odd) + [flip]


def test_scalar_multiplication(emu):
    rng = random.Random(11)
    ks = scalars()
    points = [O.G, O.hash_to_group(b"point")]
    lines, expected = [], []
    for k in ks:
        pt = points[rng.randrange(2)]
        lines.append(f"smul {h48(k)} {h48(pt[0])} {h48(pt[1])}")
        expected.append(O.serialize_element(O.mul(k, pt)).hex())
    assert run(emu, lines) == expected


def test_oprf_evaluate(emu):
    rng = random.Random(12)
    key = rng.randrange(1, O.N)
    inputs = [b"", b"\x00", rng.randbytes(12), rng.randbytes(200), rng.randbytes(65535)]
    out = run(emu, [f"eval {h48(key)} {hexb(m)}" for m in inputs])
    assert out == [O.evaluate(key.to_bytes(48, "big"), m).hex() for m in inputs]


def test_gcm_seal(emu):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    rng = random.Random(13)
    cases = [(rng.randbytes(24), rng.randbytes(12), rng.randbytes(n)) for n in (0, 1, 15, 16, 17, 31, 32, 33, 64, 1000)]
    out = run(emu, [f"seal {k.hex()} {nonce.hex()} {hexb(v)}" for k, nonce, v in cases])
    assert out == [AESGCM(k).encrypt(nonce, v, None).hex() for k, nonce, v in cases]
