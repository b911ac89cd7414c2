"""CPU checks of the plaintext-side threshold inputs (tests/plaintext_thresholds.py) at every context of its matrix and
every level.

For each constructor: the decision value recomputed from the returned input hits its target, and every constructed
input discriminates -- the oracle's result there equals what the reference's rule implies and differs from what the
opposite decision would give.  So a kernel that takes D1, D2 or D3 the wrong way at its threshold cannot match the
oracle on these inputs."""
import math
import random

import numpy as np
import pytest

import plaintext_ref as ref
import plaintext_thresholds as pt
from oracle import client_oracle as co
from oracle import oracle as orc
from oracle import pnns_oracle as pn

SIMD = [c for c in pt.CONTEXTS if pt.simd(c[1], c[3])]


def oracle_context(n, moduli, t, word_bits):
    return orc.Context(n, moduli, t, word_bits=word_bits)


def test_matrix():
    for moduli, bits, n in pt.GENERATED:
        assert moduli == orc.generate_primes([bits] * len(moduli), False, n)
    ts = {(c[3], c[4]) for c in pt.CONTEXTS}
    # both sides of the reference's one-word division switch: t^2 < 2^64 (UInt64), t^2 < 2^32 (UInt32)
    assert pt.T32_BELOW < 1 << 32 < pt.T32_ABOVE and {(pt.T32_BELOW, 64), (pt.T32_ABOVE, 64)} <= ts
    assert {(40961, 32), (65537, 32)} <= ts and 40961 < 1 << 16 < 65537
    assert (2, 64) in ts and pt.T61.bit_length() == 61 and pt.T29.bit_length() == 29
    # each is the prime = 1 mod 8192 nearest its power of two, on the side stated
    for t, lo, hi in ((pt.T32_BELOW, pt.T32_BELOW, 1 << 32), (pt.T32_ABOVE, 1 << 32, pt.T32_ABOVE),
                      (pt.T61, pt.T61, 1 << 61), (pt.T29, pt.T29, 1 << 29)):
        assert orc.is_prime(t) and t % 8192 == 1
        assert not any(orc.is_prime(v) for v in range(lo - lo % 8192 + 1, hi, 8192) if lo < v < hi)
    gamma = {64: (1 << 62) - 40797, 32: (1 << 30) - 20405}
    for _, n, moduli, t, w in pt.CONTEXTS:
        assert t < min(moduli) and t < gamma[w] and max(moduli) < 1 << (w - 2)
    assert {c[1] for c in pt.CONTEXTS} >= {16, 4096, 8192}


@pytest.mark.parametrize("name,n,moduli,t,word_bits", pt.CONTEXTS, ids=pt.IDS)
def test_translate_inputs_hit_their_targets_and_discriminate(name, n, moduli, t, word_bits):
    L = len(moduli) - 1
    rng = random.Random(t)
    for l in range(L, 0, -1):
        q = moduli[:l]
        inputs = pt.translate_inputs(moduli, t, l)
        ms = [m for m, _ in inputs]
        assert all(0 <= m < t for m in ms)
        assert {r for _, r in inputs} >= set(pt.translate_targets(t))
        assert {0, 1, t - 1} <= set(ms)
        for m, r in inputs:
            assert r == pt.translate_r(moduli, t, l, m) == math.prod(q) % t * m % t
            # the reference's one expression, in exact integers
            assert pt.translate_adjust(moduli, t, l, m) == (math.prod(q) % t * m + pt.threshold(t)) // t
            assert pt.translate_delta(moduli, t, l, m) != pt.translate_delta(moduli, t, l, m, flip=True)
        plain, where = pt.threshold_polys(ms, n, t, rng)
        zero = np.zeros((2, l, n), dtype=np.uint64)
        for k in range(len(ms)):
            got = {"ref": ref.plaintext_translate(moduli, t, zero, plain[k], ref.ADD)[0],
                   "client": co.translate_add(n, q, t, zero, plain[k])[0]}
            for p in where:
                m = int(plain[k, p])
                want, other = pt.translate_delta(moduli, t, l, m), pt.translate_delta(moduli, t, l, m, flip=True)
                for src, c0 in got.items():
                    col = [int(v) for v in c0[:, p]]
                    assert col == want and col != other, (src, l, m)
            sub = ref.plaintext_translate(moduli, t, zero, plain[k], ref.SUB)[0]
            assert np.array_equal((sub.astype(object) + got["ref"].astype(object)) % np.array(q, dtype=object)[:, None], zero[0])


@pytest.mark.parametrize("name,n,moduli,t,word_bits", pt.CONTEXTS, ids=pt.IDS)
def test_lift_inputs_hit_their_targets_and_discriminate(name, n, moduli, t, word_bits):
    o = oracle_context(n, moduli, t, word_bits)
    thr = pt.threshold(t)
    values = pt.lift_inputs(t)
    assert all(0 <= v < t for v in values) and {0, 1, t - 1} <= set(values)
    assert {thr - 1, thr} <= set(values) and (thr + 1 in values or thr + 1 == t)
    if t % 2:
        assert thr - 1 == (t - 1) // 2  # the largest value kept as is
    else:
        assert thr == t // 2            # the smallest value lifted
    plain, where = pt.threshold_polys(values, n, t, random.Random(t + 1))
    for l in range(o.L, 0, -1):
        q = moduli[:l]
        for k in range(len(values)):
            coeff = orc.ntt_inverse(n, q, o.plaintext_to_eval(plain[k], l))
            for p in where:
                v = int(plain[k, p])
                for i, qi in enumerate(q):
                    assert int(coeff[i, p]) == pt.lift_value(qi, t, v) != pt.lift_value(qi, t, v, flip=True) % qi, (l, v)


@pytest.mark.parametrize("name,n,moduli,t,word_bits", SIMD, ids=[c[0] for c in SIMD])
def test_simd_values_and_decode_eval_at_the_uncentring_threshold(name, n, moduli, t, word_bits):
    """simd_values_for_coeff encodes back to its Coeff plaintext, and decoding the Eval form of a plaintext holding
    thr - 1, thr and thr + 1 un-centres each row-0 value by the reference's rule, which differs from the opposite one."""
    o = oracle_context(n, moduli, t, word_bits)
    thr = pt.threshold(t)
    values = pt.lift_inputs(t)
    plain, where = pt.threshold_polys(values, n, t, random.Random(t + 2))
    q0 = moduli[0]
    for k in range(len(values)):
        slots = pt.simd_values_for_coeff(o, plain[k])
        assert np.array_equal(pn.encode_simd(o, slots), plain[k])
        for l in range(o.L, 0, -1):
            ev = o.plaintext_to_eval(plain[k], l)
            assert np.array_equal(ref.plaintext_to_coeff(n, q0, t, ev), plain[k]), l
            assert np.array_equal(pn.decode_simd(o, ref.plaintext_to_coeff(n, q0, t, ev)), slots), l
            row0 = orc.ntt_inverse(n, [q0], ev[0])[0]
            for p in where:
                x, v = int(row0[p]), int(plain[k, p])
                assert (x >= thr) == (v >= thr)  # a valid lift: x < thr or x >= q_0 - t + thr
                assert pt.uncentre_value(q0, t, x) == v != pt.uncentre_value(q0, t, x, flip=True), (l, v)


def test_threshold_polys_place_every_value_at_both_ends():
    for n in (16, 4096):
        values = pt.translate_targets(65537) + [5]
        plain, where = pt.threshold_polys(values, n, 65537, random.Random(n))
        assert where[0] == 0 and where[-1] == n - 1
        assert set(plain[:, 0].tolist()) == set(values) and set(plain[:, n - 1].tolist()) == set(values)
        assert set(values) <= set(plain[0, where].tolist())
