"""The noise-budget restatement (oracle/client_oracle.py) on the reference's noiseBudgetTest rules
(_TestUtilities/HeApiTestUtils.swift:1453-1485) and on the exact noise of a fresh encryption of zero."""
import math

import numpy as np
import pytest

from oracle import client_oracle as co
from oracle import oracle as orc

N = 1024


@pytest.fixture(scope="module")
def params():
    moduli = orc.generate_primes([40, 40, 41], False, N)
    t = orc.generate_primes([17], True, N)[0]
    sk = co.generate_secret_key(N, moduli, bytes(range(32)))
    return moduli, t, sk


def _add(ct, moduli):
    q = np.array([int(m) for m in moduli[:ct.shape[1]]], dtype=object)[None, :, None]
    return ((ct.astype(object) * 2) % q).astype(np.uint64)


def test_zero_ciphertext_has_infinite_budget(params):
    moduli, t, sk = params
    zero = np.zeros((2, 1, N), dtype=np.uint64)
    assert co.noise_budget(N, moduli, t, sk, zero) == math.inf
    assert co.noise_budget(N, moduli, t, sk, zero, eval_format=True) == math.inf


def test_coeff_and_eval_give_the_same_budget_and_doubling_costs_one_bit(params):
    moduli, t, sk = params
    ct_moduli = moduli[:2]
    plain = np.arange(N, dtype=np.uint64) % t
    ct = co.encrypt(N, ct_moduli, t, sk, plain, b"\x01" * 32, b"\x02" * 32)
    budget = co.noise_budget(N, moduli, t, sk, ct)
    assert budget > 0
    ev = np.stack([orc.ntt_forward(N, ct_moduli, ct[p]) for p in range(2)])
    assert co.noise_budget(N, moduli, t, sk, ev, eval_format=True) == budget
    doubled = co.noise_budget(N, moduli, t, sk, _add(ct, moduli))
    assert abs(doubled - (budget - 1)) < 0.01


def test_fresh_encryption_of_zero_has_noise_t_times_the_error(params):
    moduli, t, sk = params
    ct_moduli = moduli[:2]
    e_seed = bytes(range(100, 132))
    ct = co.encrypt(N, ct_moduli, t, sk, np.zeros(N, dtype=np.uint64), bytes(32), e_seed)
    errors = co.cbd_values(e_seed, N)
    assert co.noise_norm(N, moduli, t, sk, ct) == t * max(abs(e) for e in errors)
    q = math.prod(int(m) for m in ct_moduli)
    q_double = float(int(ct_moduli[0])) * float(int(ct_moduli[1]))
    assert co.noise_budget(N, moduli, t, sk, ct) == math.log2(q_double / (2 * float(t * max(abs(e) for e in errors))))
    assert q_double == float(q) or abs(q_double - q) / q < 1e-15


def test_secret_key_is_ternary(params):
    moduli, _, sk = params
    coeff = orc.ntt_inverse(N, moduli, sk)
    for i, q in enumerate(moduli):
        assert set(int(v) for v in coeff[i]) <= {0, 1, int(q) - 1}
    assert np.array_equal(coeff[0] == 0, coeff[2] == 0)


def test_evaluation_key_rows_are_those_of_the_whole_key():
    """generate_evaluation_key(rows=...) computes only some key ciphertexts; each has its own seeds, so they are the
    same rows of the whole key."""
    n = 64
    moduli = orc.generate_primes([40, 40, 41], False, n)
    L = len(moduli) - 1
    sk = co.generate_secret_key(n, moduli, bytes(range(32)))
    a = [bytes([i]) * 32 for i in range(3 * L)]
    e = [bytes([100 + i]) * 32 for i in range(3 * L)]
    relin, galois = co.generate_evaluation_key(n, moduli[:L], moduli[L], sk, True, [3, 2 * n - 1], a, e)
    for rows in ([1], [L - 1, 0]):
        part_relin, part_galois = co.generate_evaluation_key(n, moduli[:L], moduli[L], sk, True, [3, 2 * n - 1], a, e,
                                                             rows)
        assert np.array_equal(part_relin, relin[rows])
        for el in (3, 2 * n - 1):
            assert np.array_equal(part_galois[el], galois[el][rows])
