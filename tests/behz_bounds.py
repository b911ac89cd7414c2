"""The BEHZ multiply's magnitude bounds, in Python integers.

The GPU multiply and ct x ct inner product compute over an auxiliary base that `csrc/context.cu` picks instead of the
reference's Bsk when two conditions hold for one tensor product:

    q * B_aux > 8 N q^2            (checked as log2 B_aux >= log2 q + log2 N + 4)
    B_aux(L) * m_sk > 16 t N q     (checked as log2 B_aux(L) + log2 m_sk >= log2 t + log2 N + log2 q + 5)

`aux_base` replays that choice, `aux_pair_cap` gives the largest pair count P for which both still hold with log2 P
added to their right-hand sides (the bound past which the inner product computes over Bsk), and `fast_wrap` the
estimate P * N * t * q / 2 >= B_aux / 2 of where a sum of P worst-case products leaves the auxiliary base.

`aligned_operands` builds ciphertext pairs whose tensor products reach those bounds: every lift is +-X with
X = floor(q/2) - floor(q / 2^16), and all N terms of coefficient 0 of every product have the same sign, so
c0[0] = c2[0] = P N X^2 and c1[0] = 2 P N X^2.  `exact_floor` computes floor(t * sum D / q) for a few coefficients and
the tolerance the reference's floor allows (RnsTool.swift:378-456): approximateFloor subtracts the overflow u of the
fast base conversion of [t D]_q, a sum of L terms each below q, so u is in [0, L - 1]."""
from __future__ import annotations

import math
import random

import numpy as np

MTILDE = {64: 1 << 32, 32: 1 << 16}  # T.mTilde (Scalar.swift)
_MR_BASES = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)  # deterministic below 3.3e24


def is_prime(n: int) -> bool:
    if n < 2:
        return False
    for p in _MR_BASES:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in _MR_BASES:
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def smallest_ntt_primes(bits: int, count: int, degree: int) -> list[int]:
    """hostmath.hpp smallest_ntt_primes: the `count` smallest primes of `bits` bits that are 1 mod 2 * degree."""
    step, out = 2 * degree, []
    c, hi = (1 << (bits - 1)) + 1, 1 << bits
    while c < hi and len(out) < count:
        if c % step == 1 and is_prime(c):
            out.append(c)
        c += step
    return out


def ciphertext_moduli(moduli) -> list[int]:
    """The ciphertext moduli of a coefficient-moduli list: all but the key-switching modulus, if there is one."""
    return list(moduli[:-1]) if len(moduli) >= 2 else list(moduli)


def _slacks(n: int, moduli, t: int, pick) -> tuple[float, float]:
    # the same doubles, summed in the same order, as context.cu
    q = ciphertext_moduli(moduli)
    L = len(q)
    log_q = 0.0
    for v in q:
        log_q += math.log2(float(v))
    log_n, log_t = float(n.bit_length() - 1), math.log2(float(t))
    log_aux = log_aux_l = 0.0
    for j, v in enumerate(pick):
        log_aux += math.log2(float(v))
        if j < L:
            log_aux_l += math.log2(float(v))
    return (log_aux - (log_q + log_n + 4),
            log_aux_l + math.log2(float(pick[-1])) - (log_t + log_n + log_q + 5))


def _fast_candidates(n: int, moduli, t: int):
    """(width, primes, slack) of every auxiliary base context.cu tries, cheapest first."""
    L, nmod = len(ciphertext_moduli(moduli)), len(moduli)
    for width in (30, 55):
        cand = (smallest_ntt_primes(55, L + 1 + nmod, 1 << 31) if width == 55
                else smallest_ntt_primes(width, L + 1 + nmod, n))
        pick = [v for v in cand if v not in moduli][:L + 1]
        if len(pick) == L + 1:
            yield width, pick, min(_slacks(n, moduli, t, pick))


def aux_base(n: int, moduli, t: int, word_bits: int = 64, reference: bool = False) -> tuple[list[int], list[int]]:
    """(aux, Bsk): the base the GPU multiply computes in, and the reference's Bsk (RnsTool.swift:30-33).
    reference=True stands for HECUDA_AUX_BASE=reference."""
    L = len(ciphertext_moduli(moduli))
    bsk = smallest_ntt_primes(word_bits - 3, L + 1, n)
    if reference or word_bits != 64:
        return bsk, bsk
    for _, pick, slack in _fast_candidates(n, moduli, t):
        if slack >= 0:
            return pick, bsk
    return bsk, bsk


def aux_pair_cap(n: int, moduli, t: int, word_bits: int = 64, reference: bool = False) -> float:
    """The largest P for which both conditions hold with log2 P added to their right-hand sides: floor(2^min(slack)).
    math.inf when the multiply already computes over Bsk."""
    if reference or word_bits != 64:
        return math.inf
    for _, _, slack in _fast_candidates(n, moduli, t):
        if slack >= 0:
            return math.inf if slack >= 62 else math.floor(2.0 ** slack)
    return math.inf


def largest_fast_t(n: int, moduli) -> int:
    """The largest plaintext modulus below every ciphertext modulus for which the auxiliary base is not Bsk and is the
    same as at t = 2 (bisection: the second condition only tightens as t grows)."""
    want = aux_base(n, moduli, 2)[0]
    lo, hi = 2, min(ciphertext_moduli(moduli)) - 1
    assert want != aux_base(n, moduli, 2, reference=True)[0]
    if aux_base(n, moduli, hi)[0] == want:
        return hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if aux_base(n, moduli, mid)[0] == want else (lo, mid)
    return lo


def fast_wrap(n: int, moduli, t: int) -> int:
    """Smallest P with P N t q / 2 >= B_aux / 2: the estimate of where a sum of P aligned products leaves the auxiliary
    base (the conditions keep about 5 bits below it)."""
    q = math.prod(ciphertext_moduli(moduli))
    b = math.prod(aux_base(n, moduli, t)[0])
    return -(-b // (n * t * q))


# PredefinedRlweParameters (EncryptionParameters.swift): N, coefficient moduli (the last is the key-switching modulus
# when there are two or more), t, and the auxiliary base the multiply computes in: 30 / 55 (fast primes below 2^30 /
# h 2^32 + 1 below 2^55) or "bsk"
Q3X55 = [36028797018652673, 36028797017571329, 36028797017456641]
Q27_28_28 = [134176769, 268369921, 268361729]
Q60_60 = [1152921504606830593, 1152921504606748673]
PREDEFINED = {
    "insecure_n_16_logq_60_logt_15": (16, [1152921504606830593], 16417, 55),
    "insecure_n_512_logq_4x60_logt_20": (512, [576460752303436801, 576460752303439873, 576460752303447041,
                                               576460752303471617], 525313, 55),
    "insecure_n_8_logq_5x18_logt_5": (8, [131249, 131297, 131441, 131489, 131617], 17, 30),
    "n_4096_logq_16_33_33_logt_4": (4096, [40961, 8589852673, 8589844481], 11, 30),
    "n_4096_logq_27_28_28_logt_13": (4096, Q27_28_28, 4099, 30),
    "n_4096_logq_27_28_28_logt_16": (4096, Q27_28_28, 40961, 55),
    "n_4096_logq_27_28_28_logt_17": (4096, Q27_28_28, 65537, 55),
    "n_4096_logq_27_28_28_logt_4": (4096, Q27_28_28, 11, 30),
    "n_4096_logq_27_28_28_logt_5": (4096, Q27_28_28, 17, 30),
    "n_4096_logq_27_28_28_logt_6": (4096, Q27_28_28, 37, 30),
    "n_8192_logq_28_60_60_logt_20": (8192, [268369921] + Q60_60, 557057, 55),
    "n_8192_logq_29_60_60_logt_15": (8192, [536690689] + Q60_60, 16411, 55),
    "n_8192_logq_3x55_logt_24": (8192, Q3X55, 8404993, 55),
    "n_8192_logq_3x55_logt_29": (8192, Q3X55, 268582913, 55),
    "n_8192_logq_3x55_logt_30": (8192, Q3X55, 536903681, 55),
    "n_8192_logq_3x55_logt_42": (8192, Q3X55, 2199023288321, "bsk"),
    "n_8192_logq_40_60_60_logt_26": (8192, [1099511480321] + Q60_60, 33832961, 55),
}


def tight_shape(bits: int) -> tuple[int, list[int], int]:
    """N = 16, the three largest `bits`-bit NTT primes as coefficient moduli, and the largest t that keeps the fast
    auxiliary base: the second condition holds with less than one bit to spare."""
    n, moduli, c = 16, [], (1 << bits) - 2 * 16 + 1
    while len(moduli) < 3:
        if is_prime(c):
            moduli.append(c)
        c -= 2 * 16
    return n, moduli, largest_fast_t(n, moduli)


# ---------------------------------------------------------------------------------------------------------- operands
def aligned_x(q) -> int:
    Q = math.prod(q)
    return Q // 2 - (Q >> 16)


def lift_value(x: int, q, word_bits: int = 64) -> int:
    """liftQToQBsk of one coefficient as an integer (RnsTool.swift:324-368): the fast conversion of [m~ x]_q, then the
    small Montgomery reduction with r centred at m~ / 2."""
    mt, Q = MTILDE[word_bits], math.prod(q)
    s = sum(((mt * x) % qi * pow(Q // qi, -1, qi)) % qi * (Q // qi) for qi in q)
    r = (-s * pow(Q, -1, mt)) % mt
    if r >= mt >> 1:
        r -= mt
    v = s + Q * r
    assert v % mt == 0
    return v // mt


def residues(values, q) -> np.ndarray:
    """Integers (any shape, object or int) -> uint64 residues with a new axis of len(q) before the last axis."""
    v = np.asarray(values, dtype=object)
    out = np.stack([np.vectorize(lambda a, m=qi: a % m, otypes=[object])(v) for qi in q], axis=-2)
    return out.astype(np.uint64)


def aligned_operands(n: int, q, P: int, sign=1, rng: random.Random | None = None):
    """(lhs, rhs, signs): two (P, 2, L, N) ciphertext arrays of RNS residues and the sign of every pair.

    lhs: every coefficient of both polynomials +X.  rhs: coefficient 0 +X, coefficients 1..N-1 -X (mod q), times the
    pair's sign.  sign = +1 or -1 for every pair, or "random" (drawn from rng)."""
    Q, X = math.prod(q), aligned_x(q)
    if sign == "random":
        signs = [rng.choice((1, -1)) for _ in range(P)]
    else:
        signs = [sign] * P
    base_l = np.full(n, X, dtype=object)
    base_r = np.array([X] + [-X] * (n - 1), dtype=object)
    lhs_poly = residues(base_l % Q, q)                      # (L, N)
    rhs_poly = {s: residues((s * base_r) % Q, q) for s in (1, -1)}
    lhs = np.ascontiguousarray(np.broadcast_to(lhs_poly, (P, 2) + lhs_poly.shape))
    rhs = np.empty_like(lhs)
    for k, s in enumerate(signs):
        rhs[k, 0] = rhs[k, 1] = rhs_poly[s]
    return lhs, rhs, signs


# ------------------------------------------------------------------------------------------------------------- floor
def _crt(res, q) -> list[int]:
    """(L, N) residues -> N integers in [0, Q)."""
    Q = math.prod(q)
    out = [0] * res.shape[-1]
    for i, qi in enumerate(q):
        m = Q // qi
        f = m * pow(m, -1, qi)
        row = res[i]
        for c in range(len(out)):
            out[c] += int(row[c]) * f
    return [v % Q for v in out]


def _negacyclic_at(a, b, k: int) -> int:
    """Coefficient k of a * b mod X^N + 1 (object arrays)."""
    n = len(a)
    return int(np.dot(a[:k + 1], b[k::-1])) - (int(np.dot(a[k + 1:], b[n - 1:k:-1])) if k + 1 < n else 0)


def tensor_at(q, lhs_ct, rhs_ct, coeffs, word_bits: int = 64) -> list[list[int]]:
    """The tensor product D = lift(lhs_ct) (x) lift(rhs_ct) of one (2, L, N) ciphertext pair, as integers, at `coeffs`:
    [[D0[k] for k in coeffs], [D1[k] ...], [D2[k] ...]]."""
    lifts = {}  # aligned operands hold two values per polynomial: lift each distinct value once

    def lift(res):
        out = []
        for v in _crt(res, q):
            if v not in lifts:
                lifts[v] = lift_value(v, q, word_bits)
            out.append(lifts[v])
        return np.array(out, dtype=object)

    y = [lift(lhs_ct[p]) for p in range(2)]
    z = [lift(rhs_ct[p]) for p in range(2)]
    return [[_negacyclic_at(y[0], z[0], k) for k in coeffs],
            [_negacyclic_at(y[0], z[1], k) + _negacyclic_at(y[1], z[0], k) for k in coeffs],
            [_negacyclic_at(y[1], z[1], k) for k in coeffs]]


def exact_floor(q, t: int, lhs_ct, rhs_ct, scale: int, coeffs, word_bits: int = 64):
    """floor(t * scale * D / q) at `coeffs` for the three components of D = lift(lhs_ct) (x) lift(rhs_ct), with
    lhs_ct / rhs_ct one (2, L, N) ciphertext each: a sum of P pairs that all equal this one up to a sign has
    scale = the sum of the signs (the sum is linear, so no P N^2 terms are summed).  Returns ((3, len(coeffs))
    integers, tolerance): the reference's result r satisfies (F - r) mod q in [0, tolerance] at every sampled
    coefficient, tolerance = L - 1."""
    Q = math.prod(q)
    D = tensor_at(q, lhs_ct, rhs_ct, coeffs, word_bits)
    return [[(t * scale * d) // Q for d in row] for row in D], len(q) - 1


def within_floor(result, q, floors, tol: int, coeffs) -> bool:
    """result: (3, L, N) residues; floors from exact_floor."""
    Q = math.prod(q)
    for c in range(3):
        got = _crt(np.ascontiguousarray(result[c][:, list(coeffs)]), q)
        for F, r in zip(floors[c], got):
            if not 0 <= (F - r) % Q <= tol:
                return False
    return True


def sk_recovers(F: int, base) -> bool:
    """Whether the Shenoy-Kumaresan conversion of the floor (RnsTool.swift:402-450), given F's residues modulo the
    auxiliary base (L primes and m_sk), returns F: the exactness the second condition protects."""
    B, msk = math.prod(base[:-1]), base[-1]
    w = [(F * pow(B // b, -1, b)) % b for b in base[:-1]]
    s = sum(wi * (B // b) for wi, b in zip(w, base[:-1]))
    alpha = ((s - F) * pow(B, -1, msk)) % msk
    if alpha > msk >> 1:
        alpha -= msk
    return s - alpha * B == F
