"""GPU parity at the BFV kernels' rounding and centring thresholds (tests/threshold_inputs.py builds the inputs).

Uniform operands almost never put a decision value on its threshold (the lift's r reaches m~ / 2 once in 2^32
coefficients), so a `>` written as `>=` in a kernel passes every other parity test.  Here every column of every operand
sits at T - 1, T, T + 1 or a far value, and the results are compared bit-exactly with the oracle (budgets with ==):

  lift       behz.cu lift_kernel / lift_generic_kernel          through mulAssign, liftQToQBsk and the ct x ct inner product
  floor      behz.cu floor_kernel / floor_generic_kernel        through floorQBskToQ (a real tensor product keeps alpha
                                                                in [0, L), so only the stage entry point reaches m_sk / 2)
  decrypt    decrypt.cu scale_and_round_kernel                   through decrypt
  noise      decrypt.cu noise_norm_kernel and the norm's rounding to double   through noiseBudget
  modswitch  keyswitch.cu divround_column                        through modSwitchDown"""
import math
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
import threshold_inputs as ti
from oracle import client_oracle as co
from oracle import oracle as orc

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417, 36028797017014273]
PIR = [134176769, 268369921, 268361729]  # the PIR default moduli (27/28/28 bits), t = 17


def contexts(n, moduli, t, word_bits=64):
    g = hecuda.Context(n, moduli, t, scalar=np.uint32 if word_bits == 32 else np.uint64)
    return g, orc.Context(n, moduli, t, word_bits=word_bits)


def operands(g, seed, batch=2, word_bits=64):
    """(batch, 2, L, N) ciphertext-shaped operands whose every polynomial cycles through the lift targets."""
    q = g.ciphertextModuli
    x = ti.lift_operands(q, word_bits, g.degree, batch * 2, random.Random(seed))
    return x.reshape(batch, 2, len(q), g.degree)


# (N, coefficient moduli, t): C2 and C2-L4 (bench.py), four 62-bit ciphertext moduli (the lift's wide sums), the PIR
# moduli in a 64-bit context (30-bit auxiliary base, q_0 < m~), and 31 ciphertext moduli (lift_generic_kernel)
LIFT_SHAPES = {
    "C2": (8192, Q8192[:4], 557057),
    "C2-L4": (8192, Q8192[:5], 557057),
    "62bit-L4": (4096, None, 65537),
    "pir64": (4096, PIR, 17),
    "L31": (16, None, 97),
}


def lift_shape(name):
    n, moduli, t = LIFT_SHAPES[name]
    if name == "62bit-L4":
        moduli = orc.generate_primes([62] * 5, False, n)
    elif name == "L31":
        moduli = orc.generate_primes([60] * 32, False, n)
    return n, moduli, t


@pytest.mark.parametrize("name", list(LIFT_SHAPES))
def test_multiply_at_lift_thresholds(name):
    n, moduli, t = lift_shape(name)
    g, o = contexts(n, moduli, t)
    if name == "62bit-L4":
        L, bmax = g.L, max(g.auxModuli)
        assert bmax + L * max(g.ciphertextModuli) >= 1 << 64  # the lift's Barrett-reduced sums
    if name == "pir64":
        assert max(g.auxModuli) < 1 << 30 and min(g.ciphertextModuli) < ti.MTILDE[64]
    a, b = operands(g, 1), operands(g, 2)
    assert np.array_equal(hecuda.Bfv.mulAssign(g, a, b), o.mul(a, b))
    g.close()


def test_multiply_at_lift_thresholds_u32():
    n, t = 4096, 17
    g, o = contexts(n, PIR, t, word_bits=32)
    a, b = operands(g, 3, word_bits=32), operands(g, 4, word_bits=32)
    assert np.array_equal(hecuda.Bfv32.mulAssign(g, a.astype(np.uint32), b.astype(np.uint32)).astype(np.uint64), o.mul(a, b))
    tool = orc.RnsTool(n, g.ciphertextModuli, t, word_bits=32)
    got = hecuda.Bfv32.liftQToQBsk(g, a[0].astype(np.uint32)).astype(np.uint64)
    assert np.array_equal(got, np.stack([tool.lift(p) for p in a[0]]))
    g.close()


def test_multiply_at_lift_thresholds_reference_base(monkeypatch):
    n, moduli, t = 4096, orc.generate_primes([55] * 4, False, 4096), 557057
    monkeypatch.setenv("HECUDA_AUX_BASE", "reference")
    g, o = contexts(n, moduli, t)
    monkeypatch.delenv("HECUDA_AUX_BASE")
    assert g.auxModuli == g.bskModuli
    a, b = operands(g, 5), operands(g, 6)
    assert np.array_equal(hecuda.Bfv.mulAssign(g, a, b), o.mul(a, b))
    g.close()


@pytest.mark.parametrize("name", ["C2", "L31"])
def test_lift_stage_and_inner_product_at_lift_thresholds(name):
    """liftQToQBsk on its own (reference Bsk), and the ct x ct inner product, whose tensor_sum path lifts every pair."""
    n, moduli, t = lift_shape(name)
    g, o = contexts(n, moduli, t)
    tool = orc.RnsTool(n, g.ciphertextModuli, t)
    x = operands(g, 7, batch=1)[0]
    assert np.array_equal(hecuda.Bfv.liftQToQBsk(g, x), np.stack([tool.lift(p) for p in x]))
    lhs, rhs = operands(g, 8, batch=2)[None], operands(g, 9, batch=2)[None]
    assert np.array_equal(hecuda.Bfv.innerProductCiphertexts(g, lhs, rhs), o.inner_product(lhs, rhs))
    g.close()


# ------------------------------------------------------------------------------------------------------------ floor
@pytest.mark.parametrize("n,bits,word_bits", [(4096, [55] * 4, 64), (4096, [62] * 3, 64), (4096, None, 32),
                                              (16, [60] * 32, 64)])
def test_floor_stage_at_alpha_thresholds(n, bits, word_bits):
    moduli = PIR if bits is None else orc.generate_primes(bits, False, n)
    t = 17
    g, _ = contexts(n, moduli, t, word_bits)
    q = g.ciphertextModuli
    tool = orc.RnsTool(n, q, t, word_bits=word_bits)
    assert tool.bsk == g.bskModuli
    y = ti.floor_inputs(q, tool.bsk, n, 2, random.Random(n + len(q)))
    want = np.stack([tool.floor(p) for p in y])
    if word_bits == 32:
        got = hecuda.Bfv32.floorQBskToQ(g, y.astype(np.uint32)).astype(np.uint64)
    else:
        got = hecuda.Bfv.floorQBskToQ(g, y)
    assert np.array_equal(got, want)
    g.close()


# ---------------------------------------------------------------------------------------------------------- decrypt
@pytest.mark.parametrize("n,bits,t,word_bits", [(1024, [55, 55, 55, 55], 557057, 64), (1024, [62, 62, 62], 65537, 64),
                                                (4096, None, 17, 32)])
def test_decrypt_at_gamma_thresholds(n, bits, t, word_bits):
    moduli = PIR if bits is None else orc.generate_primes(bits, False, n)
    g, o = contexts(n, moduli, t, word_bits)
    q = g.ciphertextModuli
    assert len(q) >= 2
    sk, _ = o.keygen(11, relin=False)
    cts = ti.decrypt_ciphertexts(q, t, word_bits, n, 2, random.Random(t))
    got = hecuda.Bfv.decrypt(g, cts, sk)
    for k, ct in enumerate(cts):
        assert np.array_equal(got[k], o.decrypt(sk, ct)), k
    g.close()


# ------------------------------------------------------------------------------------------------------------ noise
def _budgets(g, sk, cts, q):
    coeff = hecuda.Bfv.noiseBudget(g, sk, cts)
    ev = np.stack([np.stack([orc.ntt_forward(g.degree, q, ct[p]) for p in range(ct.shape[0])]) for ct in cts])
    assert np.array_equal(hecuda.Bfv.noiseBudget(g, sk, ev, evalFormat=True), coeff)
    return coeff


@pytest.mark.parametrize("bits", [[17, 17, 17], [30, 30, 30], [55, 55, 55]])
def test_noise_budget_at_centring_thresholds(bits):
    """17-bit moduli keep q below 2^53, where a norm off by one changes the budget; 30 and 55 bits take two and three
    words through the kernel's wide comparisons."""
    n, t = 16, 17
    moduli = orc.generate_primes(bits + [40], False, n)
    g = hecuda.Context(n, moduli, t)
    q = g.ciphertextModuli
    sk = co.generate_secret_key(n, moduli, bytes(range(32)))
    cts, _, _ = ti.noise_ciphertexts(q, t, n, ti.noise_targets(math.prod(q)), random.Random(len(bits)))
    got = _budgets(g, sk, cts, q)
    for k, ct in enumerate(cts):
        assert got[k] == co.noise_budget(n, moduli, t, sk, ct), k
    g.close()


def test_noise_budget_rounds_the_norm_to_nearest():
    """Norms above 2^127 whose top 64 bits end in a tie and a set bit further down round up, as Double(_:) does."""
    n, t = 16, 17
    moduli = ti.ROUNDING_PRIMES + orc.generate_primes([40], False, n)
    g = hecuda.Context(n, moduli, t)
    q = g.ciphertextModuli
    sk = co.generate_secret_key(n, moduli, bytes(range(32)))
    norms = ti.rounding_norms()
    cts, _, _ = ti.noise_ciphertexts(q, t, n, norms, random.Random(2))
    got = _budgets(g, sk, cts, q)
    want = [ti.noise_budget(q, v) for v in norms]
    assert [co.noise_budget(n, moduli, t, sk, ct) for ct in cts] == want
    assert got.tolist() == want
    g.close()


# -------------------------------------------------------------------------------------------------------- modswitch
@pytest.mark.parametrize("bits", [[55, 30], [40, 55], [50, 61], [55, 62]])
def test_mod_switch_down_at_rounding_thresholds(bits):
    n, t = 4096, 17
    moduli = orc.generate_primes(bits + [56], False, n)
    g, o = contexts(n, moduli, t)
    q = g.ciphertextModuli
    assert q[-1].bit_length() == bits[-1]
    cts = ti.modswitch_ciphertexts(q, n, 2, 2, random.Random(sum(bits)))
    assert np.array_equal(hecuda.Bfv.modSwitchDown(g, cts), o.mod_switch_down(cts))
    g.close()


def test_mod_switch_down_at_rounding_thresholds_u32():
    n, t = 4096, 17
    g, o = contexts(n, PIR, t, word_bits=32)
    cts = ti.modswitch_ciphertexts(g.ciphertextModuli, n, 2, 2, random.Random(32))
    assert np.array_equal(hecuda.Bfv32.modSwitchDown(g, cts.astype(np.uint32)).astype(np.uint64), o.mod_switch_down(cts))
    g.close()
