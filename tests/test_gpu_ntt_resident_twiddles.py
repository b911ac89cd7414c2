"""The N = 8192 NTT kernels keep every twiddle in shared memory (ntt_fast.cuh, resident_twiddles): one image per modulus,
reloaded when a CTA's row changes modulus, with the odd groups of the stage with N/2 twiddles derived through
zeta = psi^(+-N/2).  Forward and inverse transforms of every modulus class, launches whose rows change modulus every
few tasks and whose task count is not a multiple of the grid, and the multiply that runs the fused forward kernel must
all stay bit-exact against the oracle."""
import numpy as np
import pytest

import hecuda
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

N = 8192
T_PLAIN = 557057


def _context(bits):
    moduli = orc.generate_primes(bits, False, N)
    return moduli, hecuda.Context(N, moduli, T_PLAIN)


def _roundtrip(g, base, row_moduli, polys, seed):
    """forward then inverse over `base` (rows_per_poly = len(row_moduli)), each checked against the oracle"""
    R = len(row_moduli)
    x = orc.fill_uniform(seed, row_moduli, N, polys * R).reshape(polys, R, N)
    x[0, :, :3] = [[0, q - 1, 1] for q in row_moduli]
    x[-1] = np.array(row_moduli, dtype=np.uint64)[:, None] - 1  # the largest residues everywhere
    fwd = hecuda.Bfv.forwardNtt(g, x, base)
    assert np.array_equal(fwd.reshape(-1, N), orc.ntt_forward(N, row_moduli, x.reshape(-1, N)))
    inv = hecuda.Bfv.inverseNtt(g, fwd, base)
    assert np.array_equal(inv, x)
    inv2 = hecuda.Bfv.inverseNtt(g, x, base)
    assert np.array_equal(inv2.reshape(-1, N), orc.ntt_inverse(N, row_moduli, x.reshape(-1, N)))


def test_every_class_including_62_bit():
    """WIDE (62-bit), MID, NARROW and SMALL ciphertext moduli, the 61-bit MID Bsk rows and the NARROW-H auxiliary rows;
    19 polynomials of 15 rows: 285 tasks, so every CTA walks rows of several moduli and the launch ends in a tail."""
    moduli, g = _context([62, 61, 58, 55, 50, 40, 30, 25])
    L = g.L
    q = moduli[:L]
    _roundtrip(g, hecuda.BASE_Q, q, 19, 1)
    _roundtrip(g, hecuda.BASE_Q_BSK, q + g.bskModuli, 19, 2)
    _roundtrip(g, hecuda.BASE_Q_AUX, q + g.auxModuli, 19, 3)


@pytest.mark.parametrize("polys", [1, 3, 5])
def test_modulus_changes_every_few_tasks(polys):
    """41 rows a polynomial over 41 different moduli (MID, NARROW, SMALL): consecutive tasks change modulus every
    `polys` tasks, so the image is reloaded between almost every two rows of a CTA (5 polynomials: 205 tasks, more than
    one wave of CTAs)."""
    bits = [61, 60, 59, 58, 57, 56, 55, 54, 53, 52, 50, 48, 45, 42, 40, 36, 33, 30, 28, 26, 25]
    moduli, g = _context(bits)
    q = moduli[:g.L]
    _roundtrip(g, hecuda.BASE_Q_BSK, q + g.bskModuli, polys, 10 + polys)


def test_narrow_h_rows_of_the_multiply():
    """[Q, aux] at C2's moduli: NARROW Q rows and NARROW-H auxiliary rows, the two-class kernels."""
    moduli, g = _context([55] * 4)
    q = moduli[:g.L]
    for p in g.auxModuli:
        assert p % (1 << 32) == 1
    _roundtrip(g, hecuda.BASE_Q_AUX, q + g.auxModuli, 67, 20)


def test_single_modulus_rows():
    """C1-8192's shape: rows of one NARROW modulus through the all-class kernels."""
    moduli, g = _context([55] * 2)
    p = moduli[0]
    x = orc.fill_uniform(30, [p], N, 300)
    fwd = hecuda.Bfv.forwardNttRows(g, p, x)
    assert np.array_equal(fwd, orc.ntt_forward(N, [p], x))
    assert np.array_equal(hecuda.Bfv.inverseNttRows(g, p, fwd), x)


@pytest.mark.parametrize("pairs", [1, 2, 67])
@pytest.mark.parametrize("nmod", [4, 5])
def test_multiply(pairs, nmod):
    """The multiply at C2's (4 moduli) and C2-L4's (5) parameters: the fused forward NTT + tensor kernel and the
    inverse both read the resident image."""
    moduli = orc.generate_primes([55] * nmod, False, N)
    g, o = hecuda.Context(N, moduli, T_PLAIN), orc.Context(N, moduli, T_PLAIN)
    L = o.L
    a = orc.fill_uniform(40 + pairs, moduli[:L], N, pairs * 2 * L).reshape(pairs, 2, L, N)
    b = orc.fill_uniform(50 + pairs, moduli[:L], N, pairs * 2 * L).reshape(pairs, 2, L, N)
    for i in range(L):  # the largest |D|: all residues q_i - 1
        a[0, :, i, :] = moduli[i] - 1
        b[0, :, i, :] = moduli[i] - 1
    assert np.array_equal(hecuda.Bfv.mulAssign(g, a, b), o.mul(a, b))
