"""CPU-side verification of the OPRF client's device code (csrc/p384.cuh, csrc/aes_gcm.cuh).

tests/emu/oprf_client_emulate.cu evaluates the same __host__ __device__ functions the client kernels call, checked
against oracle/oprf_oracle.py, tests/oprf_proof_ref.py and cryptography's AESGCM: the inverse mod n at its edges, Blind
at r = 1, n - 1 and random r, VerifyProof accepting the restatement's proofs and rejecting each tampering, unblind and
Finalize, and AES-GCM-192 open at the lengths around a block, with a tampered tag, ciphertext and key."""
import os
import random
import shutil
import subprocess

import pytest

import oprf_proof_ref as R
from oracle import oprf_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "oprf_client_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
N = O.N


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "oprf_client_emulate")
    subprocess.check_call([NVCC, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, lines):
    out = subprocess.run([binary], input="".join(line + "\n" for line in lines), capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(lines)
    return out


def h48(x: int) -> str:
    return "%096x" % x


def hx(b: bytes) -> str:
    return b.hex() or "."


def test_inverse_mod_n(emu):
    rng = random.Random(60)
    values = [1, 2, N - 1, N - 2] + [rng.randrange(1, N) for _ in range(20)]
    assert [int(x, 16) for x in run(emu, [f"ninv {h48(a)}" for a in values])] == [pow(a, -1, N) for a in values]


def test_blind(emu):
    rng = random.Random(61)
    cases = [(1, b""), (N - 1, b"keyword"), (2, b"\x00")] + \
        [(rng.randrange(1, N), rng.randbytes(rng.randrange(0, 80))) for _ in range(6)]
    out = run(emu, [f"blind {h48(r)} {hx(m)}" for r, m in cases])
    assert out == [O.blind(m, r)[1].hex() for r, m in cases]


def signed_proof(rng, key, data=None, r=None):
    """(pk bytes, query, 145-byte response) with the restatement's proof under nonce r"""
    data = rng.randbytes(12) if data is None else data
    blind_scalar = rng.randrange(1, N) if r is None else r
    query = O.blind(data, blind_scalar)[1]
    B = O.deserialize_element(query)
    D = O.mul(key, B)
    response = O.serialize_element(D) + R.generate_proof(key, rng.randrange(1, N), B, D)
    return O.serialize_element(O.mul(key, O.G)), query, response, data, blind_scalar


def flip(b: bytes, byte: int, bit: int = 0) -> bytes:
    return b[:byte] + bytes([b[byte] ^ (1 << bit)]) + b[byte + 1:]


def test_verify_accepts_and_rejects(emu):
    rng = random.Random(62)
    key = rng.randrange(1, N)
    good = [signed_proof(rng, key) for _ in range(4)]
    pk, query, response, _, _ = good[0]
    other_pk = O.serialize_element(O.mul(key + 1, O.G))
    _, other_query, other_response, _, _ = good[1]
    c_n = response[:49] + N.to_bytes(48, "big") + response[97:]
    s_n = response[:97] + N.to_bytes(48, "big")
    # D with a flipped bit: pick a bit whose flip still decodes, so the proof check itself rejects it
    flipped_d = next(f for f in (flip(response, 48, b) for b in range(8)) if _decodes(f[:49]))
    tampered = [
        (pk, query, flipped_d),                 # a flipped bit in D
        (pk, query, flip(response, 60)),        # in c
        (pk, query, flip(response, 120)),       # in s
        (pk, query, c_n),                       # c = n
        (pk, query, s_n),                       # s = n
        (other_pk, query, response),            # another key
        (pk, other_query, response),            # a response to another query
        (pk, query, other_response),            # another query's response
    ]
    lines = [f"verify {p.hex()} {q.hex()} {r.hex()}" for p, q, r, _, _ in good] + \
        [f"verify {p.hex()} {q.hex()} {r.hex()}" for p, q, r in tampered]
    assert run(emu, lines) == ["1"] * len(good) + ["0"] * len(tampered)
    # the restatement agrees on every case
    assert all(R.verify_proof(O.deserialize_element(p), O.deserialize_element(q), O.deserialize_element(r[:49]), r[49:])
               for p, q, r, _, _ in good)
    assert not any(R.verify_proof(O.deserialize_element(p), O.deserialize_element(q), O.deserialize_element(r[:49]),
                                  r[49:]) for p, q, r in tampered)


def _decodes(e: bytes) -> bool:
    try:
        O.deserialize_element(e)
        return True
    except ValueError:
        return False


def test_unblind_and_finalize(emu):
    rng = random.Random(63)
    key_bytes = rng.randrange(1, N).to_bytes(48, "big")
    cases = []
    for r, data in [(1, b""), (N - 1, b"x"), (2, rng.randbytes(100))] + \
            [(rng.randrange(1, N), rng.randbytes(rng.randrange(0, 64))) for _ in range(5)]:
        evaluated = O.blind_evaluate(key_bytes, O.blind(data, r)[1])
        cases.append((r, evaluated, data))
    out = run(emu, [f"finalize {h48(r)} {d.hex()} {hx(m)}" for r, d, m in cases])
    assert out == [O.finalize(m, r, d).hex() for r, d, m in cases]
    assert out == [O.evaluate(key_bytes, m).hex() for _, _, m in cases]


def test_open(emu):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    rng = random.Random(64)
    lines, expected = [], []
    for length in (0, 1, 15, 16, 17, 4096):
        key, nonce, value = rng.randbytes(24), rng.randbytes(12), rng.randbytes(length)
        sealed = AESGCM(key).encrypt(nonce, value, None)
        lines.append(f"open {key.hex()} {nonce.hex()} {sealed.hex()}")
        expected.append("1 " + hx(value))
        zeros = "0 " + hx(bytes(length))
        lines.append(f"open {key.hex()} {nonce.hex()} {flip(sealed, len(sealed) - 1).hex()}")  # tag
        expected.append(zeros)
        if length:
            lines.append(f"open {key.hex()} {nonce.hex()} {flip(sealed, length // 2, 3).hex()}")  # ciphertext
            expected.append(zeros)
        lines.append(f"open {flip(key, 5).hex()} {nonce.hex()} {sealed.hex()}")  # wrong key
        expected.append(zeros)
    assert run(emu, lines) == expected
