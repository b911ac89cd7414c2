"""CPU checks of the plaintext-side reference restatements (tests/plaintext_ref.py) that the GPU plaintext tests compare
against: ciphertext +- plaintext (schemeCiphertextPlaintextAdditionTest / SubtractionTest, HeApiTestUtils.swift:952-1222),
SIMD encode / decode round trips (encodingTest, :128-191) and the slot-wise product that pins the SIMD permutation."""
import random

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import pnns_oracle as pn
import plaintext_ref as ref

# (N, coefficient moduli bits, t): t = 2199023288321 (2^41 + 32769, the reference's n_8192_logq_3x55_logt_42) needs the
# 128-bit rounding term
CASES = [(64, [55, 55, 55, 55], 257), (64, [55, 55, 55, 55], 2199023288321), (128, [30, 30, 31], 40961)]


def _context(n, bits, t):
    return orc.Context(n, orc.generate_primes(bits, False, n), t)


@pytest.mark.parametrize("n,bits,t", CASES)
def test_translate_restates_the_oracle_encrypt(n, bits, t):
    """encrypt(m) = encryptZero + plaintextTranslate(Add): the restatement reproduces the oracle's own translate loop."""
    o = _context(n, bits, t)
    sk, _ = o.keygen(1, relin=False)
    rng = random.Random(n + t)
    m = np.array([rng.randrange(t) for _ in range(n)], dtype=np.uint64)
    zero = o.encrypt(7, sk, np.zeros(n, dtype=np.uint64))
    assert np.array_equal(o.encrypt(7, sk, m), ref.plaintext_translate(o.q, t, zero, m, ref.ADD))


@pytest.mark.parametrize("n,bits,t", CASES)
@pytest.mark.parametrize("polys", [2, 3])
def test_translate_decrypts_to_sum_and_difference_at_every_level(n, bits, t, polys):
    o = _context(n, bits, t)
    sk, _ = o.keygen(2, relin=False)
    rng = random.Random(3 * n + polys)
    a = np.array([rng.randrange(t) for _ in range(n)], dtype=np.uint64)
    b = np.array([rng.randrange(t) for _ in range(n)], dtype=np.uint64)
    m = np.array([rng.randrange(t) for _ in range(n)], dtype=np.uint64)
    ct = o.encrypt(11, sk, a)[None]
    if polys == 3:
        ct = o.mul(ct, o.encrypt(12, sk, b)[None])
    for _ in range(o.L):
        base = o.decrypt(sk, ct[0]).astype(object)
        mo = m.astype(object)
        want = {ref.ADD: (base + mo) % t, ref.SUB: (base - mo) % t, ref.SUB_FROM: (mo - base) % t}
        for op, expected in want.items():
            got = o.decrypt(sk, ref.plaintext_translate(o.q, t, ct[0], m, op))
            assert np.array_equal(got.astype(object), expected), (op, ct.shape)
        if ct.shape[-2] == 1:
            break
        ct = o.mod_switch_down(ct)


@pytest.mark.parametrize("n,t", [(64, 257), (64, 2199023288321), (256, 7681)])
def test_simd_round_trip_and_coeff_conversion(n, t):
    o = orc.Context(n, orc.generate_primes([55, 55, 55], False, n), t)
    rng = random.Random(n)
    for count in (n // 2, n):
        values = [rng.randrange(t) for _ in range(count)]
        plain = pn.encode_simd(o, values)
        assert pn.decode_simd(o, plain).tolist() == values + [0] * (n - count)
        for l in range(1, o.L + 1):
            assert np.array_equal(ref.plaintext_to_coeff(n, o.q[0], t, o.plaintext_to_eval(plain, l)), plain)


@pytest.mark.parametrize("n,t", [(16, 97), (64, 257)])
def test_simd_slots_multiply_pointwise(n, t):
    """The negacyclic product mod t of encode(a) and encode(b) decodes to a * b slot by slot."""
    o = orc.Context(n, orc.generate_primes([55, 55], False, n), t)
    rng = random.Random(t)
    a = [rng.randrange(t) for _ in range(n)]
    b = [rng.randrange(t) for _ in range(n)]
    prod = ref.negacyclic_mul(pn.encode_simd(o, a), pn.encode_simd(o, b), t)
    assert pn.decode_simd(o, prod).tolist() == [x * y % t for x, y in zip(a, b)]
