"""The multiply's 55-bit auxiliary base is made of primes h 2^32 + 1 (context.cu), whose NTT rows take the NARROW-H
butterflies and whose reductions take mont_reduce_h.  The product must stay the oracle's, including at the N = 8192
shapes of C2 and C2-L4, where the forward NTT, tensor product and inverse NTT run the NARROW / NARROW-H kernels."""
import numpy as np
import pytest

import hecuda
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,nmod", [(8192, 4), (8192, 5), (4096, 4), (1024, 3)])
def test_multiply_over_h_primes(n, nmod):
    moduli = orc.generate_primes([55] * nmod, False, n)
    t = 557057 if n >= 4096 else orc.generate_primes([17], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    L = nmod - 1
    assert len(g.auxModuli) == L + 1 and not set(g.auxModuli) & set(moduli)
    for p in g.auxModuli:
        assert p % (1 << 32) == 1 and (1 << 54) < p < (1 << 55)
    a = orc.fill_uniform(31, moduli[:L], n, 3 * 2 * L).reshape(3, 2, L, n)
    b = orc.fill_uniform(32, moduli[:L], n, 3 * 2 * L).reshape(3, 2, L, n)
    for i in range(L):  # the largest |D|: all residues q_i - 1
        a[0, :, i, :] = moduli[i] - 1
        b[0, :, i, :] = moduli[i] - 1
    b[1] = 0
    assert np.array_equal(hecuda.Bfv.mulAssign(g, a, b), o.mul(a, b))
