"""CPU-side verification of the OPRF server's device code (csrc/p384.cuh).

tests/emu/oprf_server_emulate.cu evaluates the same __host__ __device__ functions the server kernels call, checked
against oracle/oprf_oracle.py and tests/oprf_proof_ref.py: arithmetic mod n at its edges, the 72-byte reduction,
the per-thread recoding and constant-time ladder, decompression on both parities and every rejection, the composite
scalar, the nonce and whole 145-byte responses.  The harness takes the proof nonce r directly, so published
BlindEvaluate vectors can be pinned here."""
import hashlib
import os
import random
import shutil
import subprocess

import pytest

import oprf_proof_ref as R
from oracle import oprf_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "oprf_server_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
N = O.N


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "oprf_server_emulate")
    subprocess.check_call([NVCC, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, lines):
    out = subprocess.run([binary], input="".join(line + "\n" for line in lines), capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(lines)
    return out


def h48(x: int) -> str:
    return "%096x" % x


def test_arithmetic_mod_n(emu):
    rng = random.Random(50)
    runs = [sum(0xffffffff << (32 * i) for i in range(k)) for k in range(1, 13)]  # all-ones limb runs
    reduced = [0, 1, 2, N - 1, N - 2, N >> 1] + [v % N for v in runs] + [rng.randrange(N) for _ in range(20)]
    wide = reduced + [N, 2**384 - 1] + runs  # nmul takes any a < 2^384
    lines, expected = [], []
    for a in wide:
        for b in reduced[:10] + [rng.randrange(N)]:
            lines.append(f"nmul {h48(a)} {h48(b)}")
            expected.append(a * b % N)
    for a, b in [(a, b) for a in reduced[:12] for b in reduced[:12]] + list(zip(reduced, reversed(reduced))):
        lines += [f"nadd {h48(a)} {h48(b)}", f"nsub {h48(a)} {h48(b)}"]
        expected += [(a + b) % N, (a - b) % N]
    assert [int(x, 16) for x in run(emu, lines)] == expected


def test_reduction72_and_hash_to_scalar(emu):
    rng = random.Random(51)
    blobs = [bytes(72), b"\xff" * 72, N.to_bytes(72, "big"), (2 * N).to_bytes(72, "big"), (N - 1).to_bytes(72, "big"),
             (2**384 - 1).to_bytes(72, "big"), (N << 192).to_bytes(72, "big")] + \
        [bytes([0x80 | rng.randrange(128)]) + rng.randbytes(71) for _ in range(20)]
    assert [int(x, 16) for x in run(emu, ["nreduce72 " + b.hex() for b in blobs])] == \
        [int.from_bytes(b, "big") % N for b in blobs]
    msgs = [rng.randbytes(n) for n in (1, 48, 127, 128, 200, 300)]
    assert [int(x, 16) for x in run(emu, ["h2s " + m.hex() for m in msgs])] == [R.hash_to_scalar(m) for m in msgs]


def scalars():
    rng = random.Random(52)
    return [1, 2, 3, 4, N - 2, N - 1, N - 3, 2**200, 2**200 + 1] + [rng.randrange(1, N) for _ in range(8)]


def test_recoding_and_constant_time_ladder(emu):
    ks = scalars()
    for k, line in zip(ks, run(emu, [f"recode {h48(k)}" for k in ks])):
        odd, flip = (k, 0) if k & 1 else (N - k, 1)
        assert [int(d) for d in line.split()] == O.recode(odd) + [flip]
    rng = random.Random(53)
    points = [O.G, O.hash_to_group(b"ct")]
    lines, expected = [], []
    for k in ks:
        pt = points[rng.randrange(2)]
        lines.append(f"smulct {h48(k)} {h48(pt[0])} {h48(pt[1])}")
        expected.append(O.serialize_element(O.mul(k, pt)).hex())
    assert run(emu, lines) == expected


def test_decompression(emu):
    rng = random.Random(54)
    valid = [O.serialize_element(O.mul(rng.randrange(1, N), O.G)) for _ in range(12)]
    assert {v[0] for v in valid} == {2, 3}
    for v, line in zip(valid, run(emu, ["decompress " + v.hex() for v in valid])):
        x, y = O.deserialize_element(v)
        assert line.split() == [h48(x), h48(y)]
    off_curve = next(x for x in range(1, 100) if not O.is_square((x ** 3 + O.A * x + O.B) % O.P))
    invalid = [b"\0" + valid[0][1:], b"\1" + valid[0][1:], b"\4" + valid[0][1:], b"\2" + O.P.to_bytes(48, "big"),
               b"\3" + (O.P + 1).to_bytes(48, "big"), b"\2" + (2**384 - 1).to_bytes(48, "big"),
               b"\2" + off_curve.to_bytes(48, "big"), bytes(49)]
    assert run(emu, ["decompress " + v.hex() for v in invalid]) == ["invalid"] * len(invalid)


def test_composite_nonce_and_responses(emu):
    rng = random.Random(55)
    key = rng.randrange(1, N)
    pk = O.mul(key, O.G)
    seed48 = hashlib.sha384(R._framed(O.serialize_element(pk)) + R._framed(R.SEED_DST)).digest()
    queries = [O.blind(rng.randbytes(10), rng.randrange(1, N))[1] for _ in range(4)]
    evaluated = [O.serialize_element(O.mul(key, O.deserialize_element(q))) for q in queries]
    out = run(emu, [f"composite {seed48.hex()} {q.hex()} {d.hex()}" for q, d in zip(queries, evaluated)])
    expected = [R.hash_to_scalar(R._framed(seed48) + b"\0\0" + R._framed(q) + R._framed(d) + b"Composite")
                for q, d in zip(queries, evaluated)]
    assert [int(x, 16) for x in out] == expected
    seed32 = rng.randbytes(32)
    assert [int(x, 16) for x in run(emu, [f"nonce {h48(key)} {seed32.hex()} {q.hex()}" for q in queries])] == \
        [R.proof_nonce(key, seed32, q) for q in queries]
    rs = [1, 2, N - 1, rng.randrange(1, N)]
    out = run(emu, [f"prove {h48(key)} {h48(r)} {q.hex()}" for r, q in zip(rs, queries)])
    assert out == [(d + R.generate_proof(key, r, O.deserialize_element(q), O.deserialize_element(d))).hex()
                   for r, q, d in zip(rs, queries, evaluated)]
    keys = [1, 2, N - 1, key]
    out = run(emu, [f"respond {h48(k)} {seed32.hex()} {q.hex()}" for k, q in zip(keys, queries)] +
              [f"respond {h48(key)} {seed32.hex()} {bytes(49).hex()}"])
    assert out == [R.blind_evaluate_verifiable(k.to_bytes(48, "big"), q, seed32).hex()
                   for k, q in zip(keys, queries)] + ["invalid"]
