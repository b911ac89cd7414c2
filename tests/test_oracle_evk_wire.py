"""Seeded evaluation keys on the oracle side (tests/evk_wire_ref.py): a re-seeded key still relinearizes and applies
Galois automorphisms correctly, and its serialized poly0 plus the seed expand back to the key."""
import numpy as np
import pytest

import evk_wire_ref as ref
from oracle import oracle as orc

TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)


@pytest.mark.parametrize("n,bits,t", [(16, TEST_MODULI_BITS, 1153), (64, [55, 55, 55], 65537)])
def test_reseeded_keys_switch_and_expand_back(n, bits, t):
    o = orc.Context(n, orc.generate_primes(bits, False, n), t)
    rng = np.random.default_rng(n)
    sk, relin = o.keygen(3)
    element = 2 * n - 1
    galois = o.galois_keygen(4, sk, element)
    relin_seeds, galois_seeds = ref.random_seeds(rng, o.L), ref.random_seeds(rng, o.L)
    relin2, relin_wire = ref.reseed_key(o, sk, relin, relin_seeds)
    galois2, galois_wire = ref.reseed_key(o, sk, galois, galois_seeds)
    assert not np.array_equal(relin2[:, 1], relin[:, 1])
    for key, wire, seeds in ((relin2, relin_wire, relin_seeds), (galois2, galois_wire, galois_seeds)):
        for i in range(o.L):
            assert np.array_equal(ref.expand_seeded_key_ciphertext(o, wire[i].tobytes(), seeds[i].tobytes()), key[i])

    m1 = rng.integers(0, t, size=n, dtype=np.uint64)
    m2 = rng.integers(0, t, size=n, dtype=np.uint64)
    ct1, ct2 = o.encrypt(11, sk, m1), o.encrypt(12, sk, m2)
    ct3 = o.mul(ct1, ct2)[0]
    want = o.decrypt(sk, ct3)
    assert np.array_equal(o.decrypt(sk, o.relinearize(ct3, relin)[0]), want)
    assert np.array_equal(o.decrypt(sk, o.relinearize(ct3, relin2)[0]), want)
    rotated = o.apply_galois(ct1, element, galois2)[0]
    assert np.array_equal(o.decrypt(sk, rotated), orc.galois_coeff(n, [t], element, m1.reshape(1, n)).reshape(n))
    assert np.array_equal(o.decrypt(sk, rotated), o.decrypt(sk, o.apply_galois(ct1, element, galois)[0]))
