"""Exact restatements of the reference's plaintext-side steps for the plaintext tests (test infrastructure only).

  plaintext_translate   plaintextTranslate, Bfv+Encrypt.swift:75-139 (+ HeScheme.subCoeff = plaintext + -ciphertext,
                        HeScheme.swift:1540-1542): poly 0 gets +- [floor(Q/t) m + floor(([Q]_t m + ceil(t/2)) / t)]_{q_i}
  plaintext_to_coeff    Plaintext.convertToCoeffFormat, Plaintext.swift:176-194

Big-integer arithmetic throughout, so every t (including t > 2^32, where the rounding term needs 128 bits) is exact.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import oracle as orc

ADD, SUB, SUB_FROM = 0, 1, 2


def translate_delta(q, t: int, plain) -> list:
    """Per row i of Q = q_0..q_{l-1}: [floor(Q/t) m + floor(([Q]_t m + tThreshold) / t)]_{q_i} for each coefficient m."""
    Q = math.prod(int(v) for v in q)
    m = np.asarray(plain, dtype=np.uint64).astype(object)
    v = m * (Q // t) + (m * (Q % t) + (t + 1) // 2) // t
    return [np.array(v % int(qi), dtype=np.uint64) for qi in q]


def plaintext_translate(q, t: int, ct, plain, op: int) -> np.ndarray:
    """One Coeff ciphertext (polys, l, N) with moduli q[:l] and one Coeff plaintext (N,) -> the translated ciphertext."""
    c = np.array(ct, dtype=np.uint64)
    l = c.shape[1]
    rows = translate_delta([int(v) for v in q[:l]], t, plain)
    for i in range(l):
        qi = np.uint64(q[i])
        x, d = c[0, i], rows[i]
        if op == ADD:
            c[0, i] = (x + d) % qi
        elif op == SUB:
            c[0, i] = (x + qi - d) % qi
        else:
            c[0, i] = (d + qi - x) % qi
            for k in range(1, c.shape[0]):
                c[k, i] = (qi - c[k, i]) % qi
    return c


def plaintext_to_coeff(n: int, q0: int, t: int, eval_plain) -> np.ndarray:
    """Row 0 of an Eval plaintext -> inverse NTT mod q_0 -> x >= tThreshold ? x - (q_0 - t) : x."""
    row = orc.ntt_inverse(n, [q0], np.asarray(eval_plain, dtype=np.uint64).reshape(-1, n)[0])[0]
    return np.where(row >= np.uint64((t + 1) // 2), row - np.uint64(q0 - t), row).astype(np.uint64)


def negacyclic_mul(a, b, t: int) -> np.ndarray:
    """Schoolbook product in Z_t[X]/(X^N + 1)."""
    a = [int(v) for v in a]
    b = [int(v) for v in b]
    n = len(a)
    out = [0] * n
    for i, x in enumerate(a):
        if x == 0:
            continue
        for j, y in enumerate(b):
            k = i + j
            if k < n:
                out[k] += x * y
            else:
                out[k - n] -= x * y
    return np.array([v % t for v in out], dtype=np.uint64)
