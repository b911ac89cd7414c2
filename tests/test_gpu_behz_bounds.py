"""GPU parity of the BEHZ multiply and the ct x ct inner product at their magnitude bounds (tests/behz_bounds.py).

Every lift of the aligned operands is +-(q/2 - q/2^16) and all N terms of coefficient 0 of each product have the same
sign, so the tensor product and the floor reach their worst case instead of a random walk about sqrt(N) below it.  The
multiply runs at the reference's predefined parameter sets with their own t, at shapes whose t sits on the auxiliary
base's second condition, over Bsk, at UInt32 and at L = 31.  The inner product runs across aux_max_pairs, the pair
count past which it leaves the auxiliary base for Bsk, up to four times where the auxiliary base would wrap.  Results
are compared bit-exactly with the oracle (which computes over the reference's Bsk), and on sampled coefficients with
floor(t * sum D / q) within the floor's tolerance."""
import math
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import behz_bounds as bb
import hecuda
from oracle import oracle as orc

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417, 36028797017014273]
MUL_SETS = ["n_8192_logq_3x55_logt_24", "n_8192_logq_3x55_logt_29", "n_8192_logq_3x55_logt_30",
            "n_8192_logq_3x55_logt_42", "n_8192_logq_28_60_60_logt_20", "n_8192_logq_29_60_60_logt_15",
            "n_8192_logq_40_60_60_logt_26", "n_4096_logq_27_28_28_logt_5", "n_4096_logq_27_28_28_logt_13"]


def shape(name):
    """(N, coefficient moduli, t) of a predefined set, a tight-margin shape ("tight30", "tight52", and "+1" for the
    next t, which leaves that base), or L = 31 (32 moduli of 60 bits: the generic lift and floor)."""
    if name in bb.PREDEFINED:
        return bb.PREDEFINED[name][:3]
    if name.startswith("tight"):
        n, moduli, t = bb.tight_shape(int(name[5:7]))
        return n, moduli, t + 1 if name.endswith("+1") else t
    assert name == "L31"
    return 16, orc.generate_primes([60] * 32, False, 16), 97


def both_signs(n, q):
    """(2, 2, L, N) x 2: one aligned pair with sign +1, one with sign -1, as a batch of two multiplies."""
    pos, neg = bb.aligned_operands(n, q, 1, 1), bb.aligned_operands(n, q, 1, -1)
    return np.concatenate([pos[0], neg[0]]), np.concatenate([pos[1], neg[1]])


def check_floor(got, q, t, lhs, rhs, scale=1, word_bits=64):
    coeffs = sorted({0, 1, got.shape[-1] // 2, got.shape[-1] - 1})
    F, tol = bb.exact_floor(q, t, lhs, rhs, scale, coeffs, word_bits)
    assert bb.within_floor(got, q, F, tol, coeffs)


def check_multiply(g, o, n, q, t, word_bits=64):
    a, b = both_signs(n, q)
    if word_bits == 32:
        got = hecuda.Bfv32.mulAssign(g, a.astype(np.uint32), b.astype(np.uint32)).astype(np.uint64)
    else:
        got = hecuda.Bfv.mulAssign(g, a, b)
    assert np.array_equal(got, o.mul(a, b))
    for k in range(2):
        check_floor(got[k], q, t, a[k], b[k], word_bits=word_bits)


# --------------------------------------------------------------------------------------------------------- multiply
@pytest.mark.parametrize("name", MUL_SETS + ["tight30", "tight30+1", "tight52", "tight52+1", "L31"])
def test_multiply_at_aligned_operands(name):
    n, moduli, t = shape(name)
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    assert g.auxModuli == bb.aux_base(n, moduli, t)[0]
    check_multiply(g, o, n, g.ciphertextModuli, t)
    g.close()


@pytest.mark.parametrize("name", ["n_8192_logq_3x55_logt_30", "tight52"])
def test_multiply_at_aligned_operands_reference_base(monkeypatch, name):
    n, moduli, t = shape(name)
    monkeypatch.setenv("HECUDA_AUX_BASE", "reference")
    g = hecuda.Context(n, moduli, t)
    monkeypatch.delenv("HECUDA_AUX_BASE")
    assert g.auxModuli == g.bskModuli == bb.aux_base(n, moduli, t, reference=True)[0]
    check_multiply(g, orc.Context(n, moduli, t), n, g.ciphertextModuli, t)
    g.close()


def test_multiply_at_aligned_operands_u32():
    n, moduli, t = shape("n_4096_logq_27_28_28_logt_5")
    g, o = hecuda.Context(n, moduli, t, scalar=np.uint32), orc.Context(n, moduli, t, word_bits=32)
    assert g.auxModuli == bb.aux_base(n, moduli, t, word_bits=32)[0]
    check_multiply(g, o, n, g.ciphertextModuli, t, word_bits=32)
    g.close()


@pytest.mark.parametrize("mod_switch", [False, True])
def test_mul_relinearize_at_aligned_operands(mod_switch):
    n, moduli, t = 8192, Q8192[:4], 557057  # C2
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    assert g.auxModuli == bb.aux_base(n, moduli, t)[0]
    _, rk = o.keygen(3)
    key = hecuda.EvaluationKey(g, rk)
    a, b = both_signs(n, g.ciphertextModuli)
    want = o.relinearize(o.mul(a, b), rk)
    if mod_switch:
        want = o.mod_switch_down(want)
    assert np.array_equal(hecuda.Bfv.mulRelinearize(g, a, b, key, modSwitchDown=mod_switch), want)
    g.close()


# ---------------------------------------------------------------------------------------------------- inner product
def sign_groups(n, q, P, seed):
    """(3, P, 2, L, N) x 2 and the signs: all pairs +1, all -1, random signs."""
    groups = [bb.aligned_operands(n, q, P, s, random.Random(seed)) for s in (1, -1, "random")]
    return (np.stack([x[0] for x in groups]), np.stack([x[1] for x in groups]), [x[2] for x in groups])


def check_groups(got, q, t, lhs, rhs, signs):
    for k, s in enumerate(signs):
        pos = [i for i, v in enumerate(s) if v > 0]
        i0 = pos[0] if pos else 0  # every pair equals this one up to its sign
        check_floor(got[k], q, t, lhs[k, i0], rhs[k, i0], scale=sum(s) * s[i0])


def pair_counts(n, moduli, t):
    cap, wrap = bb.aux_pair_cap(n, moduli, t), bb.fast_wrap(n, moduli, t)
    return sorted({1, 2, cap, cap + 1, 2 * wrap, 4 * wrap})


@pytest.mark.parametrize("name", ["tight30", "tight52"])
def test_inner_product_across_the_pair_bound(name):
    n, moduli, t = shape(name)
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    q = g.ciphertextModuli
    assert g.auxModuli == bb.aux_base(n, moduli, t)[0] != g.bskModuli
    for P in pair_counts(n, moduli, t):
        lhs, rhs, signs = sign_groups(n, q, P, P)
        got = hecuda.Bfv.innerProductCiphertexts(g, lhs, rhs)
        assert np.array_equal(got, o.inner_product(lhs, rhs)), P
        check_groups(got, q, t, lhs, rhs, signs)
    g.close()


def test_inner_product_at_n_8192_logq_3x55_logt_30():
    """1040 pairs, just past where the 55-bit auxiliary base would wrap (about 1024).  Device memory: the inputs and
    (4P + 3)(2L + 1)N words of scratch, about 2 GB."""
    n, moduli, t = shape("n_8192_logq_3x55_logt_30")
    P = 1040
    assert bb.aux_pair_cap(n, moduli, t) < bb.fast_wrap(n, moduli, t) < P
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    q = g.ciphertextModuli
    lhs, rhs, signs = bb.aligned_operands(n, q, P, 1)
    got = hecuda.Bfv.innerProductCiphertexts(g, lhs[None], rhs[None])
    assert np.array_equal(got, o.inner_product(lhs[None], rhs[None]))
    check_floor(got[0], q, t, lhs[0], rhs[0], scale=P)
    g.close()


def test_inner_product_device_entry_point_past_the_pair_bound():
    n, moduli, t = shape("tight30")
    P = 4 * bb.fast_wrap(n, moduli, t)
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    q = g.ciphertextModuli
    lhs, rhs, signs = sign_groups(n, q, P, 7)
    a, b = torch.from_numpy(lhs.view(np.int64)).cuda(), torch.from_numpy(rhs.view(np.int64)).cuda()
    out = torch.empty((3, 3, len(q), n), dtype=torch.int64, device="cuda")
    rc = hecuda.load_library().hecuda_bfv_inner_product_device(g._h, a.data_ptr(), b.data_ptr(), out.data_ptr(), P, 3, None)
    torch.cuda.synchronize()
    assert rc == 0
    got = out.cpu().numpy().view(np.uint64)
    assert np.array_equal(got, o.inner_product(lhs, rhs))
    check_groups(got, q, t, lhs, rhs, signs)
    g.close()
