"""The multiply's inverse NTT folds the floor's first step, y_i = [x_i (Q/q_i)^-1]_{q_i}, into its last-stage constants
(kScaleTMontFloor, context.hpp), the floor's row constants carry (B/b_k)^-1 (FloorConsts), and the lift and floor
give each CTA one column tile and lift both operands in one launch (behz.cu).  Products must stay the oracle's: batches of many tiles, N below one tile, the ct x ct inner
product (tensor_sum path), and moduli whose lazy sums take the wide-sum path (Barrett reductions on MID / WIDE rows)."""
import numpy as np
import pytest

import hecuda
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _operands(seed, moduli, n, batch, L):
    a = orc.fill_uniform(seed, moduli[:L], n, batch * 2 * L).reshape(batch, 2, L, n)
    b = orc.fill_uniform(seed + 1, moduli[:L], n, batch * 2 * L).reshape(batch, 2, L, n)
    for i in range(L):  # the largest |D|: all residues q_i - 1
        a[0, :, i, :] = moduli[i] - 1
        b[0, :, i, :] = moduli[i] - 1
    a[1, 0] = 0
    return a, b


@pytest.mark.parametrize("n,bits,nmod,batch", [(8192, 55, 4, 24), (8192, 55, 5, 8), (4096, 55, 4, 48), (4096, 62, 6, 12),
                                               (2048, 61, 3, 64), (64, 60, 3, 7), (16, 55, 3, 5)])
def test_multiply_with_folded_floor_scaling(n, bits, nmod, batch):
    moduli = orc.generate_primes([bits] * nmod, False, n)
    t = 557057 if n >= 4096 else orc.generate_primes([12], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    a, b = _operands(41, moduli, n, batch, o.L)
    assert np.array_equal(hecuda.Bfv.mulAssign(g, a, b), o.mul(a, b))


@pytest.mark.parametrize("n,bits,nmod,pairs,groups", [(4096, 55, 4, 8, 6), (8192, 55, 4, 3, 4), (1024, 62, 6, 4, 3)])
def test_ct_ct_inner_product_with_folded_floor_scaling(n, bits, nmod, pairs, groups):
    moduli = orc.generate_primes([bits] * nmod, False, n)
    t = orc.generate_primes([12], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    L = o.L
    lhs = orc.fill_uniform(5, moduli[:L], n, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, n)
    rhs = orc.fill_uniform(6, moduli[:L], n, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, n)
    for i in range(L):
        lhs[0, 0, :, i, :] = moduli[i] - 1
        rhs[0, 0, :, i, :] = moduli[i] - 1
    assert np.array_equal(hecuda.Bfv.innerProductCiphertexts(g, lhs, rhs), o.inner_product(lhs, rhs))
