"""Inputs that put the plaintext side's rounding and centring decisions exactly on their thresholds.

Three decisions compare a value derived from one plaintext coefficient with a threshold:

  D1 translate  plaintextTranslate (Bfv+Encrypt.swift)      adjust = floor(([Q_l]_t m + tThreshold) / t), i.e. a carry
                                                            iff r = [[Q_l]_t m]_t >= t - tThreshold = floor(t / 2)
  D2 lift       convertToEvalFormat (Plaintext.swift)       v < tThreshold ? v : v + (q_r - t)
  D3 uncentre   convertToCoeffFormat (Plaintext.swift)      x >= tThreshold ? x - (q_0 - t) : x, on row 0 after the
                                                            inverse NTT mod q_0

with tThreshold = (t + 1) // 2 (RnsTool.swift).  A uniform m < t reaches one given r with probability 1 / t, so for
t above a few thousand the random-input tests never put D1 on its threshold; D2 and D3 likewise.  The constructors
here solve for the inputs in Python ints and return the decision value next to each one; `flip=True` gives a
decision's result taken the other way round, which the tests show differs.

D3 is only fed valid lifts: row 0 of the Eval form of a plaintext coefficient v is v (v < tThreshold) or
v + q_0 - t, never a value in [tThreshold, q_0 - t + tThreshold).  So a `>=` written as `>` in the un-centring, which
only changes the result at x = tThreshold, gives the same result on every valid plaintext.

CONTEXTS is the parameter matrix the CPU and GPU tests share: t on both sides of the reference's one-word division
switch (t^2 < 2^64 for UInt64, t^2 < 2^32 for UInt32), the predefined sets' t, t = 2 and a 61-bit t.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import pnns_oracle as pn

# (id, N, coefficient moduli [q_0 .. q_{L-1}, q_ks], t, word bits).  Moduli not taken from a predefined set are
# orc.generate_primes(bits, False, N), listed in GENERATED (test_plaintext_thresholds.py checks they still are).
PIR = [134176769, 268369921, 268361729]                                       # n_4096_logq_27_28_28
Q8192_55 = [36028797018652673, 36028797017571329, 36028797017456641]          # n_8192_logq_3x55_logt_42
Q8192_33 = [1099511480321, 1152921504606830593, 1152921504606748673]          # the t = 33832961 set
Q16_50 = [1125899906842273, 1125899906842177, 1125899906841377, 1125899906840897]                    # 4 x 50 bits
Q4096_55 = [36028797018652673, 36028797018529793, 36028797018267649, 36028797017939969]              # 4 x 55 bits
Q4096_62 = [4611686018427322369, 4611686018427289601, 4611686018427215873, 4611686018427199489]      # 4 x 62 bits
Q4096_30 = [1073692673, 1073668097, 1073651713, 1073643521]                                          # 4 x 30 bits
T32_BELOW = 4294828033       # the largest prime = 1 mod 8192 below 2^32
T32_ABOVE = 4294991873       # the smallest prime = 1 mod 8192 above 2^32
T61 = 2305843009213554689    # the largest prime = 1 mod 8192 below 2^61: below every 62-bit q_i and gamma = 2^62 - 40797
T29 = 536813569              # the largest prime = 1 mod 8192 below 2^29: below every 30-bit q_i and gamma = 2^30 - 20405
GENERATED = [(Q16_50, 50, 16), (Q4096_55, 55, 4096), (Q4096_62, 62, 4096), (Q4096_30, 30, 4096)]  # (moduli, bits, N)
CONTEXTS = [
    ("t2-n16", 16, Q16_50, 2, 64),
    ("t97-n16", 16, Q16_50, 97, 64),
    ("t17-n4096", 4096, PIR, 17, 64),
    ("t65537-n4096", 4096, PIR, 65537, 64),
    ("t4294828033-n4096", 4096, Q4096_55, T32_BELOW, 64),
    ("t4294991873-n4096", 4096, Q4096_55, T32_ABOVE, 64),
    ("t33832961-n8192", 8192, Q8192_33, 33832961, 64),
    ("t2199023288321-n8192", 8192, Q8192_55, 2199023288321, 64),
    ("t2305843009213554689-n4096", 4096, Q4096_62, T61, 64),
    ("u32-t40961-n4096", 4096, PIR, 40961, 32),
    ("u32-t65537-n4096", 4096, PIR, 65537, 32),
    ("u32-t536813569-n4096", 4096, Q4096_30, T29, 32),
]
IDS = [c[0] for c in CONTEXTS]


def simd(n: int, t: int) -> bool:
    """Context.supportsSimdEncoding: t is a prime = 1 mod 2N (t in CONTEXTS is 2 or a prime)."""
    return t > 2 and (t - 1) % (2 * n) == 0


def threshold(t: int) -> int:
    """RnsTool.tThreshold."""
    return (t + 1) // 2


def _unique(values, t: int):
    out = []
    for v in values:
        if 0 <= v < t and v not in out:
            out.append(v)
    return out


# -------------------------------------------------------------------------------------------------------- D1 translate
def translate_targets(t: int):
    """r around the carry threshold floor(t / 2), and the far values 0, 1, t - 1 (those below t, without repeats)."""
    h = t // 2
    return _unique([h - 1, h, h + 1, 0, 1, t - 1], t)


def translate_r(q, t: int, l: int, m: int) -> int:
    """D1's decision value for coefficient m at level l: r = [[Q_l]_t m]_t."""
    return math.prod(q[:l]) % t * m % t


def translate_adjust(q, t: int, l: int, m: int, flip: bool = False) -> int:
    """plaintextTranslate's adjust = floor([Q_l]_t m / t) + (r >= floor(t / 2)) (the other way round with flip)."""
    w = math.prod(q[:l]) % t
    carry = (w * m % t >= t - threshold(t)) != flip
    return w * m // t + carry


def translate_delta(q, t: int, l: int, m: int, flip: bool = False):
    """The value plaintextTranslate adds to row i of c0: [floor(Q_l / t) m + adjust]_{q_i}, i < l."""
    v = math.prod(q[:l]) // t * m + translate_adjust(q, t, l, m, flip)
    return [v % qi for qi in q[:l]]


def translate_inputs(q, t: int, l: int):
    """[(m, r)]: plaintext coefficients m whose r = [[Q_l]_t m]_t is each translate target, m = r [Q_l]_t^-1 mod t
    ([Q_l]_t is invertible: every prime factor of Q_l is a q_i > t), then the far coefficients 0, 1, t - 1."""
    w = math.prod(q[:l]) % t
    w_inv = pow(w, -1, t)
    ms = _unique([r * w_inv % t for r in translate_targets(t)] + [0, 1, t - 1], t)
    return [(m, w * m % t) for m in ms]


# ------------------------------------------------------------------------------------------------------------ D2 lift
def lift_inputs(t: int):
    """Coeff values around tThreshold = (t + 1) // 2, and 0, 1, t - 1.  For odd t, tThreshold - 1 = (t - 1) / 2 is the
    largest value kept as is; for even t, tThreshold = t / 2 is the smallest one lifted."""
    thr = threshold(t)
    return _unique([thr - 1, thr, thr + 1, 0, 1, t - 1], t)


def lift_value(qi: int, t: int, v: int, flip: bool = False) -> int:
    """convertToEvalFormat's centred lift of v into Z_{q_i} (before the NTT), the other way round with flip."""
    keep = (v < threshold(t)) != flip
    return v if keep else v + qi - t


# -------------------------------------------------------------------------------------------------------- D3 uncentre
def uncentre_value(q0: int, t: int, x: int, flip: bool = False) -> int:
    """convertToCoeffFormat's un-centring of a row-0 Coeff value x, as an integer (negative when the opposite decision
    takes x below q_0 - t), the other way round with flip."""
    sub = (x >= threshold(t)) != flip
    return x - (q0 - t) if sub else x


def simd_values_for_coeff(ctx, coeff) -> np.ndarray:
    """The slot values whose encodeSimd is the Coeff plaintext `coeff`: decodeSimd of it (forward NTT mod t, then the
    encoding permutation).  ctx: an oracle Context whose t supports SIMD encoding."""
    return pn.decode_simd(ctx, np.asarray(coeff, dtype=np.uint64))


# ------------------------------------------------------------------------------------------------------- placement
def spots(n: int, count: int):
    """`count` positions (at most N) spread over [0, N - 1], including 0 and N - 1."""
    count = max(2, min(n, count))
    return sorted({round(i * (n - 1) / (count - 1)) for i in range(count)})


def threshold_polys(values, n: int, t: int, rng, copies: int = 3):
    """(len(values), N) plaintexts.  Polynomial k holds values[(i + k) % V] at spot i of spots(N, V * copies), and a
    uniform value below t everywhere else.  So every value sits at position 0 in one polynomial and at N - 1 in another,
    and polynomial 0 holds every value at least once.  Returns (plaintexts, spot positions)."""
    V = len(values)
    where = spots(n, V * copies)
    out = np.array([[rng.randrange(t) for _ in range(n)] for _ in range(V)], dtype=np.uint64)
    for k in range(V):
        for i, p in enumerate(where):
            out[k, p] = values[(i + k) % V]
    return out, where
