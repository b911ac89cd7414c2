"""CPU checks of the threshold inputs (tests/threshold_inputs.py) and of the noise norm's rounding to double.

For every constructor: the decision value recomputed from its definition hits its target in every column, and every
column discriminates -- the oracle's result equals what the reference's rule implies there and differs from what the
opposite decision would give.  So a kernel that takes one of these decisions the wrong way at its threshold cannot
match the oracle on these inputs.

wide_to_double (csrc/hostmath.hpp), which turns the noise budget's multi-word infinity norm into a double, is compiled
into a small host program and compared with Python's float(int) (correctly rounded, ties to even) at exact ties with
and without bits below them, with the leading word's top bit set and clear, at 2 to 8 words."""
import math
import os
import random
import shutil
import struct
import subprocess

import numpy as np
import pytest

import threshold_inputs as ti
from oracle import client_oracle as co
from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = shutil.which("g++") or shutil.which("c++")
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417, 36028797017014273]
PIR = [134176769, 268369921, 268361729]  # the PIR default moduli (27/28/28 bits), t = 17
N = 16


def columns(a):
    """(rows, n) -> the n columns as lists of ints."""
    return [[int(v) for v in a[:, j]] for j in range(a.shape[1])]


# (ciphertext moduli, word bits): C2's, 62-bit wide sums, q_0 below m~ in 64 bits, Bfv<UInt32>, one modulus, L > 16
LIFT_CASES = {
    "c2": (Q8192[:3], 64),
    "62bit": (orc.generate_primes([62] * 4, False, N), 64),
    "pir64": (PIR[:2], 64),
    "pir32": (PIR[:2], 32),
    "one": (Q8192[:1], 64),
    "l31": (orc.generate_primes([60] * 31, False, N), 64),
}


@pytest.mark.parametrize("case", list(LIFT_CASES))
def test_lift_inputs(case):
    q, wb = LIFT_CASES[case]
    rng = random.Random(case)
    polys = 2
    x = ti.lift_operands(q, wb, N, polys, rng)
    tool = orc.RnsTool(x.shape[-1], q, 17, word_bits=wb)
    mt = ti.MTILDE[wb]
    assert mt >> 1 in ti.lift_targets(wb)
    for k in range(polys):
        lifted = tool.lift(x[k])
        assert np.array_equal(lifted[: len(q)], x[k])
        for j, col in enumerate(columns(x[k])):
            assert ti.lift_r(q, wb, col) == ti.lift_targets(wb)[(j + k) % 6]
            bsk = [int(v) for v in lifted[len(q):, j]]
            assert bsk == ti.lift_bsk(q, tool.bsk, wb, col), (k, j)
            assert bsk != ti.lift_bsk(q, tool.bsk, wb, col, flip=True), (k, j)


def test_lift_target_out_of_reach_is_refused():
    """One modulus below m~ reaches only q_0 of the 2^32 values of r: the constructor says so instead of looping."""
    with pytest.raises(ValueError):
        ti.lift_operands(PIR[:1], 64, 6, 1, random.Random(0))


@pytest.mark.parametrize("q,wb", [(Q8192[:3], 64), (orc.generate_primes([62] * 3, False, N), 64), (PIR[:2], 32),
                                  (orc.generate_primes([60] * 17, False, N), 64)])
def test_floor_inputs(q, wb):
    rng = random.Random(len(q) * wb)
    tool = orc.RnsTool(N, q, 17, word_bits=wb)
    msk = tool.bsk[-1]
    polys = 2
    y = ti.floor_inputs(q, tool.bsk, N, polys, rng)
    for k in range(polys):
        floored = tool.floor(y[k])
        for j, col in enumerate(columns(y[k])):
            assert ti.floor_alpha(q, tool.bsk, col) == ti.floor_targets(msk)[(j + k) % 6]
            got = [int(v) for v in floored[:, j]]
            assert got == ti.floor_q(q, tool.bsk, col), (k, j)
            assert got != ti.floor_q(q, tool.bsk, col, flip=True), (k, j)


@pytest.mark.parametrize("q,t,wb", [(Q8192[:3], 557057, 64), (orc.generate_primes([62] * 2, False, N), 65537, 64),
                                    (PIR, 17, 32)])
def test_decrypt_inputs(q, t, wb):
    rng = random.Random(t)
    cts = ti.decrypt_ciphertexts(q, t, wb, N, 3, rng)
    assert not cts[:, 1].any()
    tool = orc.RnsTool(N, q, t, word_bits=wb)
    o = orc.Context(N, list(q) + orc.generate_primes([60 if wb == 64 else 29], False, N), t, word_bits=wb)
    sk, _ = o.keygen(3, relin=False)
    signs = set()
    for k, ct in enumerate(cts):
        out = tool.scale_and_round(ct[0])
        assert np.array_equal(o.decrypt(sk, ct), out)
        for j, col in enumerate(columns(ct[0])):
            assert ti.decrypt_mod_gamma(q, t, wb, col) == ti.decrypt_targets(wb)[(j + k) % 6]
            want, sign = ti.decrypt_value(q, t, wb, col)
            assert int(out[j]) == want, (k, j)
            assert ti.decrypt_value(q, t, wb, col, flip=True)[0] != want, (k, j)
            signs.add(sign)
    assert signs == {True, False}  # polyModT - sGamma wraps in some columns and not in others


def _noise_key(n, moduli):
    return co.generate_secret_key(n, moduli, bytes(range(32)))


@pytest.mark.parametrize("bits", [[17, 17, 17], [25, 25], [30, 30, 30], [55, 55, 55]])
def test_noise_inputs(bits):
    """Three moduli of 17 bits keep q below 2^53, so the budget is exact and a norm off by one changes it; the wider
    sets reach two and three words, where only the norm itself tells the decisions apart."""
    moduli = orc.generate_primes(bits + [40], False, N)
    q, t = moduli[:-1], 17
    Q = math.prod(q)
    sk = _noise_key(N, moduli)
    values = ti.noise_targets(Q)
    cts, composed, where = ti.noise_ciphertexts(q, t, N, values, random.Random(Q))
    for k, ct in enumerate(cts):
        assert composed[k][where[k]] == values[k]
        norm = co.noise_norm(N, moduli, t, sk, ct)
        assert norm == ti.noise_norm(Q, composed[k])
        flipped = ti.noise_norm(Q, composed[k], flip_at=where[k])
        assert norm != flipped, k
        budget = co.noise_budget(N, moduli, t, sk, ct)
        assert budget == ti.noise_budget(q, norm)
        if Q < 1 << 53:
            assert budget != ti.noise_budget(q, flipped), k
        ev = np.stack([orc.ntt_forward(N, q, ct[p]) for p in range(2)])
        assert co.noise_budget(N, moduli, t, sk, ev, eval_format=True) == budget


def test_noise_rounding_inputs():
    """Norms above 2^127 whose top 64 bits end in a tie with a set bit below: the budget uses the norm rounded up."""
    q = ti.ROUNDING_PRIMES
    moduli = q + orc.generate_primes([40], False, N)
    Q = math.prod(q)
    assert 1 << 128 < Q < 1 << 129 and all(p % 64 == 1 for p in q)
    sk = _noise_key(N, moduli)
    norms = ti.rounding_norms()
    cts, composed, where = ti.noise_ciphertexts(q, 17, N, norms, random.Random(1))
    for k, ct in enumerate(cts):
        assert co.noise_norm(N, moduli, 17, sk, ct) == norms[k] <= (Q + 1) >> 1
        budget = co.noise_budget(N, moduli, 17, sk, ct)
        top = norms[k] >> 64  # the leading 64 bits; the tie rounded to even instead of up
        truncated = math.log2(math.prod(float(p) for p in q) / (2 * math.ldexp(float(top & ~0x7FF), 64)))
        assert budget == ti.noise_budget(q, norms[k]) and budget != truncated


@pytest.mark.parametrize("bits", [[55, 30], [55, 55], [50, 61], [40, 55, 62], [27, 28]])
def test_modswitch_inputs(bits):
    q = orc.generate_primes(bits, False, N)
    rng = random.Random(sum(bits))
    cts = ti.modswitch_ciphertexts(q, N, 2, 2, rng)
    targets = ti.modswitch_targets(q[-1])
    for k in range(2):
        for p in range(2):
            x = cts[k, p]
            out = orc.divide_round_qlast(N, q, x)
            for j, col in enumerate(columns(x)):
                assert col[-1] == targets[(j + k * 2 + p) % 5]
                got = [int(v) for v in out[:, j]]
                assert got == ti.modswitch_value(q, col), (k, p, j)
                assert got != ti.modswitch_value(q, col, flip=True), (k, p, j)


# ------------------------------------------------------------------------------------------------- wide_to_double
@pytest.fixture(scope="module")
def wide_to_double(tmp_path_factory):
    if CXX is None:
        pytest.skip("no C++ compiler")
    binary = str(tmp_path_factory.mktemp("wide") / "wide_to_double")
    subprocess.check_call([CXX, "-O2", "-std=c++17", "-o", binary, os.path.join(ROOT, "tests", "emu", "wide_to_double.cpp")])

    def run(values):
        """values: (x, words) pairs -> the doubles the host function returns."""
        lines = []
        for x, w in values:
            words = [(x >> (64 * i)) & ((1 << 64) - 1) for i in range(w)]
            assert sum(v << (64 * i) for i, v in enumerate(words)) == x
            lines.append(" ".join(str(v) for v in [w] + words))
        out = subprocess.run([binary], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return [struct.unpack("<d", struct.pack("<Q", int(v)))[0] for v in out.split()]

    return run


def _ties(w, lz, rng):
    """Values of `w` words whose leading word has `lz` leading zeros and whose leading 64 bits end in an exact tie
    (the bit below the 53-bit mantissa set, the ten below it clear), with nothing, one bit just below, one bit at the
    bottom, or random bits below the leading 64; both parities of the mantissa."""
    low = 64 * w - lz - 64  # bit position of the leading window's lowest bit
    out = []
    for lsb in (0, 1):
        mant = (1 << 52) | (rng.getrandbits(51) << 1) | lsb
        window = (mant << 11) | (1 << 10)
        for below in (0, 1 << (low - 1), 1, rng.getrandbits(low) | 1):
            out.append((window << low) | below)
    return out


@pytest.mark.parametrize("w", range(2, 9))
def test_wide_to_double_rounds_like_float(wide_to_double, w):
    rng = random.Random(w)
    values = []
    for lz in (0, 1, 11, 63):
        values += [(x, w) for x in _ties(w, lz, rng)]
    if w >= 3:
        # a zero word right below the leading word, the tie decided by a bit further down
        for lz in (0, 5):
            top = ((1 << 63) >> lz) | (1 << (10 - lz) if lz <= 10 else 0)
            for below in (0, 1, 1 << (64 * (w - 2) - 1)):
                values.append(((top << (64 * (w - 1))) | below, w))
    # exact values, random values, and leading zero words
    values += [(0, w), (1, w), ((1 << 53) + 1, w), ((1 << 64) - 1, w), (1 << 64, w), ((1 << 64) + 1, w)]
    values += [(rng.getrandbits(64 * w - rng.randrange(64 * w - 1)), w) for _ in range(200)]
    values += [(x, w + 2) for x, _ in values[:20]]
    got = wide_to_double(values)
    for (x, words), d in zip(values, got):
        assert d == float(x), (hex(x), words, d, float(x))


def test_wide_to_double_reported_case(wide_to_double):
    """x = 2^127 + 2^74 + 1 over two words: the tie in the top word is broken by the low word, so it rounds up."""
    x = (((1 << 63) | 0x400) << 64) | 1
    assert wide_to_double([(x, 2)]) == [float(x)] == [1.7014118346046927e+38]
