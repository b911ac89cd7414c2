"""Inputs that put the BFV kernels' rounding and centring decisions exactly on their thresholds.

Each decision below compares one value with a threshold T.  A `>` written as `>=` changes the result for the one value
T, which a uniform input reaches with probability about 1/T (2^-32 for the lift's r in Bfv<UInt64>, about 2^-60 for the
floor's alpha).  The constructors here solve, column by column, for inputs whose decision value is T - 1, T, T + 1 or a
far value (0, 1, m - 1), following the reference's definitions in Python ints:

  lift       smallMontgomeryReduce (RnsTool.swift)      r = [(sum_i z_i Q/q_i) (-Q^-1)]_m~, kept iff r < m~ >> 1
  floor      convertApproximateBskToQ (RnsTool.swift)   alpha centred iff alpha > m_sk >> 1
  decrypt    scaleAndRound (RnsTool.swift)              the gamma correction iff [.]_gamma > gamma / 2
  noise      noiseBudgetEval (Bfv+Decrypt.swift)        coeff > (q + 1) >> 1 counts as q - coeff
  modswitch  divideAndRoundQLast (PolyRq.swift)         the last residue x rounds up iff x > floor(q_l / 2)

Next to each constructor is the decision value recomputed from its definition and the result the reference's rule
implies; `flip=True` gives the result with that one decision taken the other way, which the tests show differs.
"""
from __future__ import annotations

import math

import numpy as np

MTILDE = {64: 1 << 32, 32: 1 << 16}                         # T.mTilde, Scalar.swift
GAMMA = {64: (1 << 62) - 40797, 32: (1 << 30) - 20405}      # T.rnsCorrectionFactor, Scalar.swift


def around(threshold: int, modulus: int):
    """threshold - 1, threshold, threshold + 1 and the far values 0, 1, modulus - 1."""
    return [threshold - 1, threshold, threshold + 1, 0, 1, modulus - 1]


def _punctured(q):
    Q = math.prod(q)
    return Q, [Q // qi for qi in q]


def _target(targets, poly: int, col: int) -> int:
    """Column `col` of polynomial `poly` takes one target; the targets cycle along the columns, shifted per polynomial."""
    return targets[(col + poly) % len(targets)]


# ------------------------------------------------------------------------------------------------------------- lift
def lift_targets(word_bits: int):
    mt = MTILDE[word_bits]
    return around(mt >> 1, mt)


def lift_r(q, word_bits: int, column) -> int:
    """r of smallMontgomeryReduce for one column (x_0 .. x_{L-1}): z_i = [x_i [m~]_{q_i} (Q/q_i)^-1]_{q_i},
    r = [(sum_i z_i Q/q_i) (-Q^-1)]_m~."""
    mt = MTILDE[word_bits]
    Q, P = _punctured(q)
    z = [int(x) * mt * pow(p, -1, qi) % qi for x, p, qi in zip(column, P, q)]
    return sum(zi * p for zi, p in zip(z, P)) * -pow(Q, -1, mt) % mt


def lift_bsk(q, bsk, word_bits: int, column, flip: bool = False):
    """The Bsk rows of liftQToQBsk for one column: y = (x~ + Q r_c) / m~ mod b_j, with r_c = r if r < m~ >> 1 else
    r - m~ (the other way round with flip)."""
    mt = MTILDE[word_bits]
    Q, P = _punctured(q)
    z = [int(x) * mt * pow(p, -1, qi) % qi for x, p, qi in zip(column, P, q)]
    x_tilde = sum(zi * p for zi, p in zip(z, P))
    r = x_tilde * -pow(Q, -1, mt) % mt
    keep = r < mt >> 1
    r_c = r if keep != flip else r - mt
    y, rem = divmod(x_tilde + Q * r_c, mt)
    assert rem == 0
    return [y % b for b in bsk]


def lift_operands(q, word_bits: int, n: int, polys: int, rng) -> np.ndarray:
    """(polys, L, n) Coeff residues whose column j of polynomial k has r = lift_targets[(j + k) % 6].  x_1 .. x_{L-1}
    are random; z_0 is solved modulo m~ (Q/q_0 is odd, so invertible), lifted to z_0 + k m~ < q_0 and mapped back to
    x_0.  When q_0 < m~ the random residues are redrawn until the solution fits."""
    mt = MTILDE[word_bits]
    L = len(q)
    Q, P = _punctured(q)
    w = [mt * pow(p, -1, qi) % qi for p, qi in zip(P, q)]  # x_i -> z_i
    w0_inv = pow(w[0], -1, q[0])
    p0_inv = pow(P[0], -1, mt)
    targets = lift_targets(word_bits)
    out = np.empty((polys, L, n), dtype=np.uint64)
    for k in range(polys):
        for j in range(n):
            c = _target(targets, k, j)
            while True:
                x = [0] + [rng.randrange(qi) for qi in q[1:]]
                rest = sum(xi * wi % qi * p for xi, wi, qi, p in zip(x[1:], w[1:], q[1:], P[1:]))
                z0 = (-c * Q - rest) * p0_inv % mt
                if z0 < q[0]:
                    break
                if L == 1:
                    raise ValueError(f"r = {c} is out of reach: q_0 < m~ and no other residue to vary")
            z0 += rng.randrange((q[0] - 1 - z0) // mt + 1) * mt
            x[0] = z0 * w0_inv % q[0]
            out[k, :, j] = x
    return out


# ------------------------------------------------------------------------------------------------------------ floor
def floor_targets(msk: int):
    return around(msk >> 1, msk)


def _floor_parts(q, bsk, column):
    """approximateFloor and the conversion products: (w_0 .. w_{L-1}, f_msk, [sum_i w_i B/b_i]_{m_sk})."""
    L = len(q)
    B, msk = bsk[:L], bsk[L]
    Q, P = _punctured(q)
    y = [int(x) * pow(p, -1, qi) % qi for x, p, qi in zip(column[:L], P, q)]
    fbc = sum(yi * p for yi, p in zip(y, P))  # fast base conversion of x_Q, before reduction
    f = [(int(column[L + j]) - fbc) * pow(Q, -1, b) % b for j, b in enumerate(bsk)]
    Bp, PB = _punctured(B)
    w = [fj * pow(pb, -1, b) % b for fj, pb, b in zip(f[:L], PB, B)]
    return w, f[L], sum(wi * pb for wi, pb in zip(w, PB)) % msk, Bp, PB


def floor_alpha(q, bsk, column) -> int:
    """alpha_sk of convertApproximateBskToQ for one column over [Q, Bsk]: [(sum_i w_i B/b_i - f_msk) B^-1]_{m_sk}."""
    msk = bsk[len(q)]
    _, f_msk, alpha0, Bp, _ = _floor_parts(q, bsk, column)
    return (alpha0 - f_msk) * pow(Bp, -1, msk) % msk


def floor_q(q, bsk, column, flip: bool = False):
    """floorQBskToQ for one column: [sum_i w_i B/b_i - alpha_c B]_{q_i}, alpha_c = alpha if alpha <= m_sk >> 1 else
    alpha - m_sk (the other way round with flip)."""
    msk = bsk[len(q)]
    w, f_msk, alpha0, Bp, PB = _floor_parts(q, bsk, column)
    alpha = (alpha0 - f_msk) * pow(Bp, -1, msk) % msk
    centred = alpha > msk >> 1
    alpha_c = alpha - msk if centred != flip else alpha
    s = sum(wi * pb for wi, pb in zip(w, PB))
    return [(s - alpha_c * Bp) % qi for qi in q]


def floor_inputs(q, bsk, n: int, polys: int, rng) -> np.ndarray:
    """(polys, 2L+1, n) residues over [Q, Bsk] whose column j of polynomial k has alpha = floor_targets[(j + k) % 6]:
    the Q and B rows are random and the m_sk row is solved (f_msk is x_msk Q^-1 minus a function of the Q rows)."""
    L = len(q)
    msk = bsk[L]
    Q, P = _punctured(q)
    targets = floor_targets(msk)
    out = np.empty((polys, 2 * L + 1, n), dtype=np.uint64)
    for k in range(polys):
        for j in range(n):
            col = [rng.randrange(m) for m in list(q) + list(bsk)]
            col[2 * L] = 0
            _, _, alpha0, Bp, _ = _floor_parts(q, bsk, col)
            f_msk = (alpha0 - _target(targets, k, j) * Bp) % msk
            y = [x * pow(p, -1, qi) % qi for x, p, qi in zip(col[:L], P, q)]
            col[2 * L] = (f_msk * Q + sum(yi * p for yi, p in zip(y, P))) % msk
            out[k, :, j] = col
    return out


# ---------------------------------------------------------------------------------------------------------- decrypt
def decrypt_targets(word_bits: int):
    g = GAMMA[word_bits]
    return around(g // 2, g)


def _decrypt_sums(q, t: int, word_bits: int, column):
    g = GAMMA[word_bits]
    Q, P = _punctured(q)
    y = [int(c) * (g * t % qi) * pow(p, -1, qi) % qi for c, p, qi in zip(column, P, q)]
    s = sum(yi * p for yi, p in zip(y, P))
    return s * -pow(Q, -1, t) % t, s * -pow(Q, -1, g) % g


def decrypt_mod_gamma(q, t: int, word_bits: int, column) -> int:
    """[v gamma t]_Q converted to gamma and times -Q^-1 (scaleAndRound's polyModGamma) for one column v."""
    return _decrypt_sums(q, t, word_bits, column)[1]


def decrypt_value(q, t: int, word_bits: int, column, flip: bool = False):
    """scaleAndRound (scaling factor 1) for one column: (plaintext coefficient, whether polyModT >= sGamma).  sGamma is
    -(gamma - polyModGamma) mod t if polyModGamma > gamma / 2, else polyModGamma mod t (the other way round with flip)."""
    g = GAMMA[word_bits]
    mod_t, mod_g = _decrypt_sums(q, t, word_bits, column)
    greater = (mod_g > g // 2) != flip
    s = -(g - mod_g) % t if greater else mod_g % t
    return (mod_t - s) * pow(g, -1, t) % t, mod_t >= s


def decrypt_ciphertexts(q, t: int, word_bits: int, n: int, count: int, rng) -> np.ndarray:
    """(count, 2, L, n) Coeff ciphertexts with c1 = 0, so that c0 s^0 = c0 whatever the secret key, whose column j of
    ciphertext k has polyModGamma = decrypt_targets[(j + k) % 6].  y_1 .. y_{L-1} are random, y_0 is solved modulo gamma
    and kept when it is below q_0 (probability about q_0 / gamma per draw); needs L >= 2."""
    g = GAMMA[word_bits]
    L = len(q)
    if L < 2:
        raise ValueError("the gamma targets need two moduli or more")
    Q, P = _punctured(q)
    to_c = [pow((g * t % qi) * pow(p, -1, qi) % qi, -1, qi) for p, qi in zip(P, q)]  # y_i -> c0_i
    p0_inv = pow(P[0], -1, g)
    targets = decrypt_targets(word_bits)
    out = np.zeros((count, 2, L, n), dtype=np.uint64)
    for k in range(count):
        for j in range(n):
            c = _target(targets, k, j)
            while True:
                y = [0] + [rng.randrange(qi) for qi in q[1:]]
                y[0] = (-c * Q - sum(yi * p for yi, p in zip(y[1:], P[1:]))) * p0_inv % g
                if y[0] < q[0]:
                    break
            out[k, 0, :, j] = [yi * ci % qi for yi, ci, qi in zip(y, to_c, q)]
    return out


# ------------------------------------------------------------------------------------------------------------ noise
def noise_targets(Q: int):
    """Values of [v t]_Q around the centring threshold (Q + 1) >> 1, and the far values 1 and Q - 1."""
    half = (Q + 1) >> 1
    return [half - 1, half, half + 1, 1, Q - 1]


def noise_norm(Q: int, values, flip_at=None) -> int:
    """noiseBudgetEval's infinity norm of the composed coefficients `values`: coeff > (Q + 1) >> 1 counts as Q - coeff.
    flip_at: the index of one coefficient whose decision is taken the other way round."""
    half = (Q + 1) >> 1
    norms = [(Q - v if v > half else v) if i != flip_at else (v if v > half else Q - v) for i, v in enumerate(values)]
    return max(norms)


def noise_ciphertexts(q, t: int, n: int, values, rng, small_bits: int = 20):
    """One (2, L, n) Coeff ciphertext per value V, as an array (len(values), 2, L, n): c1 = 0 and c0 = [t^-1 V]_Q at one
    column (so [v t]_Q = V there, whatever the secret key), and [v t]_Q random below 2^small_bits in magnitude at the
    others.  Returns (ciphertexts, composed [v t]_Q of every column, the column holding V)."""
    Q = math.prod(q)
    t_inv = pow(t, -1, Q)
    out = np.zeros((len(values), 2, len(q), n), dtype=np.uint64)
    composed, where = [], []
    for k, V in enumerate(values):
        col = (5 * k + 3) % n
        vs = [rng.randrange(-(1 << small_bits), 1 << small_bits) % Q for _ in range(n)]
        vs[col] = V % Q
        for j, v in enumerate(vs):
            c0 = v * t_inv % Q
            out[k, 0, :, j] = [c0 % qi for qi in q]
        composed.append(vs)
        where.append(col)
    return out, composed, where


def noise_budget(q, norm: int) -> float:
    """log2(qDouble / (2 norm)) with qDouble the product of the moduli as doubles, in order, and Double(norm) rounded to
    nearest (Bfv+Decrypt.swift:137-146)."""
    if norm == 0:
        return math.inf
    q_double = 1.0
    for qi in q:
        q_double *= float(qi)
    return math.log2(q_double / (2 * float(norm)))


# The norm rounding case: three NTT primes (1 mod 64, so N <= 32) whose product is just above 2^128, and norms whose top
# 64 bits end in an exact tie with a set bit far below: Double(_:) rounds them up.
ROUNDING_PRIMES = [0x6597FA95601, 0x6597FA95641, 0x6597FA959C1]


def rounding_norms(ks=(0, 1, 7, 1234, 3999)):
    return [((1 << 63 | 0x400 | k << 12) << 64) | 1 for k in ks]


# -------------------------------------------------------------------------------------------------------- modswitch
def modswitch_targets(q_last: int):
    h = q_last // 2
    return [h - 1, h, h + 1, 0, q_last - 1]


def modswitch_value(q, column, flip: bool = False):
    """divideAndRoundQLast for one column: (x_i - r) q_l^-1 mod q_i with r = x_l if x_l <= floor(q_l / 2) else
    x_l - q_l (the other way round with flip)."""
    ql = q[-1]
    x = int(column[-1])
    r = x if (x <= ql // 2) != flip else x - ql
    return [(int(c) - r) * pow(ql, -1, qi) % qi for c, qi in zip(column[:-1], q[:-1])]


def modswitch_ciphertexts(q, n: int, count: int, polys: int, rng) -> np.ndarray:
    """(count, polys, l, n) residues: random rows, the last row cycling through modswitch_targets."""
    targets = modswitch_targets(q[-1])
    out = np.empty((count, polys, len(q), n), dtype=np.uint64)
    for k in range(count):
        for p in range(polys):
            for i, qi in enumerate(q[:-1]):
                out[k, p, i] = [rng.randrange(qi) for _ in range(n)]
            out[k, p, -1] = [_target(targets, k * polys + p, j) for j in range(n)]
    return out
