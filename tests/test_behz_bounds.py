"""CPU checks of tests/behz_bounds.py: the aligned operands reach the multiply's worst case, the oracle (over the
reference's 61-bit Bsk) stays exact there far past where the GPU's auxiliary base would wrap, and the base choice at
every predefined parameter set."""
import math
import random

import numpy as np
import pytest

import behz_bounds as bb
from oracle import oracle as orc

PREDEFINED, Q3X55, Q27_28_28 = bb.PREDEFINED, bb.Q3X55, bb.Q27_28_28
COEFFS = lambda n: sorted({0, 1, n // 2, n - 1})  # noqa: E731


tight_shape = bb.tight_shape


@pytest.mark.parametrize("name", list(PREDEFINED))
def test_aux_base_at_predefined_sets(name):
    n, moduli, t, want = PREDEFINED[name]
    aux, bsk = bb.aux_base(n, moduli, t)
    q = bb.ciphertext_moduli(moduli)
    assert bsk == orc.RnsTool(n, q, t).bsk
    if want == "bsk":
        assert aux == bsk and bb.aux_pair_cap(n, moduli, t) == math.inf
    else:
        assert aux != bsk and max(aux).bit_length() == want and len(aux) == len(q) + 1
        assert not set(aux) & set(moduli)
        assert bb.aux_pair_cap(n, moduli, t) >= 1  # math.inf when the slack is 62 bits or more
    assert bb.aux_base(n, moduli, t, reference=True) == (bsk, bsk)


def test_aux_base_at_n_8192_logq_3x55():
    """logt_42's t fails the second condition and falls back to Bsk; the cap of the others halves with every bit of t."""
    caps = {}
    for logt in (24, 29, 30):
        n, moduli, t, _ = PREDEFINED[f"n_8192_logq_3x55_logt_{logt}"]
        caps[logt] = bb.aux_pair_cap(n, moduli, t)
        assert bb.aux_base(n, moduli, t)[0] == bb.smallest_ntt_primes(55, 3, 1 << 31)
    assert caps[30] < caps[29] < caps[24]
    n, moduli, t, _ = PREDEFINED["n_8192_logq_3x55_logt_42"]
    assert bb.fast_wrap(n, moduli, t) == 65536  # over Bsk


@pytest.mark.parametrize("bits", [30, 52])
def test_tight_shape_sits_on_the_second_condition(bits):
    n, moduli, t = tight_shape(bits)
    aux, bsk = bb.aux_base(n, moduli, t)
    assert aux != bsk and max(aux).bit_length() == (30 if bits == 30 else 55)
    assert bb.aux_base(n, moduli, t + 1)[0] != aux
    assert bb.aux_pair_cap(n, moduli, t) == 1
    assert 32 <= bb.fast_wrap(n, moduli, t) <= 33


@pytest.mark.parametrize("n,moduli,word_bits", [(16, orc.generate_primes([30] * 3, False, 16), 64),
                                                (8192, Q3X55, 64), (4096, Q27_28_28, 32),
                                                (16, orc.generate_primes([60] * 32, False, 16), 64)])
def test_aligned_operands_reach_the_worst_case(n, moduli, word_bits):
    q = bb.ciphertext_moduli(moduli)
    Q, X = math.prod(q), bb.aligned_x(q)
    assert bb.lift_value(X, q, word_bits) == X and bb.lift_value(Q - X, q, word_bits) == -X
    for sign in (1, -1):
        lhs, rhs, signs = bb.aligned_operands(n, q, 2, sign)
        assert signs == [sign, sign] and lhs.shape == (2, 2, len(q), n) and lhs.dtype == np.uint64
        D = bb.tensor_at(q, lhs[0], rhs[0], [0, 1, n - 1], word_bits)
        assert D[0][0] == D[2][0] == sign * n * X * X and D[1][0] == sign * 2 * n * X * X
        assert all(abs(d) < abs(row[0]) for row in D for d in row[1:])  # coefficient 0 is the largest
        P = 5
        F, tol = bb.exact_floor(q, 7, lhs[0], rhs[0], P, [0], word_bits)
        assert F[1][0] == (7 * sign * 2 * P * n * X * X) // Q and tol == len(q) - 1


def test_fast_base_wraps_where_the_estimate_says():
    """The Shenoy-Kumaresan step over the fast base, replayed in integers at coefficient 0 of c1: exact up to the cap
    and past it up to about fast_wrap, wrong from there on.  Over Bsk it stays exact."""
    for n, moduli, t in (tight_shape(30), tight_shape(52), (8192, Q3X55, 536903681), (8192, Q3X55, 268582913)):
        q = bb.ciphertext_moduli(moduli)
        Q, X = math.prod(q), bb.aligned_x(q)
        aux, bsk = bb.aux_base(n, moduli, t)
        cap, wrap = bb.aux_pair_cap(n, moduli, t), bb.fast_wrap(n, moduli, t)
        for sign in (1, -1):
            F = lambda P: (t * sign * P * 2 * n * X * X) // Q  # noqa: E731
            assert bb.sk_recovers(F(cap), aux)
            assert 16 * cap <= wrap
            first = next(P for P in range(cap, 4 * wrap) if not bb.sk_recovers(F(P), aux))
            assert wrap - 2 <= first <= wrap + 2, (n, t, first, wrap)
            assert bb.sk_recovers(F(4 * wrap), bsk)


@pytest.mark.parametrize("bits", [30, 52])
def test_oracle_inner_product_is_exact_far_past_the_fast_wrap(bits):
    n, moduli, t = tight_shape(bits)
    q = bb.ciphertext_moduli(moduli)
    o = orc.Context(n, moduli, t)
    wrap = bb.fast_wrap(n, moduli, t)
    rng = random.Random(bits)
    for P in (1, wrap, 4 * wrap, 16 * wrap):
        for sign in (1, -1, "random"):
            lhs, rhs, signs = bb.aligned_operands(n, q, P, sign, rng)
            got = o.inner_product(lhs[None], rhs[None])[0]
            pos = [k for k, s in enumerate(signs) if s > 0]
            k0 = pos[0] if pos else 0  # every pair is this one up to its sign
            scale = sum(signs) * signs[k0]
            F, tol = bb.exact_floor(q, t, lhs[k0], rhs[k0], scale, COEFFS(n))
            assert bb.within_floor(got, q, F, tol, COEFFS(n)), (P, sign)


@pytest.mark.parametrize("name", ["n_8192_logq_3x55_logt_42", "n_8192_logq_40_60_60_logt_26",
                                  "n_4096_logq_27_28_28_logt_13"])
def test_oracle_multiply_is_exact_at_aligned_operands(name):
    n, moduli, t, _ = PREDEFINED[name]
    q = bb.ciphertext_moduli(moduli)
    o = orc.Context(n, moduli, t)
    for sign in (1, -1):
        lhs, rhs, _ = bb.aligned_operands(n, q, 1, sign)
        got = o.mul(lhs, rhs)[0]
        F, tol = bb.exact_floor(q, t, lhs[0], rhs[0], 1, COEFFS(n))
        assert bb.within_floor(got, q, F, tol, COEFFS(n)), sign
