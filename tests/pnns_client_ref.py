"""Exact restatement of the reference's PNNS client for the client tests (test infrastructure only).

Reference code followed (paths relative to Sources/):

  * normalizedScaledAndRounded   PrivateNearestNeighborSearch/Util.swift:74-89
  * Array2d.mul(_:modulus:)      Util.swift:99-123 (the centred modular product)
  * fixedPointCosineSimilarity   Util.swift:141-159
  * maxScalingFactor             Config.swift:112-120
  * Client.generateQuery/decrypt Client.swift:73-127
  * CrtComposer.compose          HomomorphicEncryption/CrtComposer.swift:76-97
  * getDatabaseForTesting        _TestUtilities/PnnsUtilities/PnnsUtils.swift:37-45

Float arithmetic is numpy float32 scalar steps, each rounded once, the sums left to right -- what Swift's Float does.
The packing, SIMD coding and encryption are those of oracle/pnns_oracle.py and oracle/client_oracle.py.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import client_oracle as co
from oracle import pnns_oracle as opn

F32 = np.float32


def float32_of_int(v: int) -> np.float32:
    """Float(v) for an integer: round to nearest, ties to even (exact also past 2^53)."""
    v = int(v)
    mag = abs(v)
    if mag < 1 << 53:
        return F32(float(v))
    shift = mag.bit_length() - 24
    q, r = divmod(mag, 1 << shift)
    half = 1 << (shift - 1)
    if r > half or (r == half and q & 1):
        q += 1
    return F32(float(q << shift) * (1 if v > 0 else -1))


def normalized_scaled_and_rounded(rows, scaling_factor) -> list:
    """Array2d.normalizedScaledAndRounded (Util.swift:74-89) into Int64: raises ValueError where Swift traps."""
    out = []
    for row, scaled in zip(rows, _rescale(rows, scaling_factor)):
        if any(not np.isfinite(F32(x)) for x in row):
            raise ValueError("not finite")
        out.append([v if isinstance(v, int) else _round_away(v) for v in scaled])
    return out


def _rescale(rows, scaling_factor):
    """(value * s) / norm per value as float32 (0 marks a zero-norm row as int 0)."""
    s = F32(scaling_factor)
    out = []
    with np.errstate(all="ignore"):
        for row in rows:
            row = [F32(x) for x in row]
            total = F32(0)
            for x in row:
                total = F32(total + F32(x * x))
            norm = F32(np.sqrt(total))
            out.append([0 if norm == 0 else F32(F32(x * s) / norm) for x in row])
    return out


def _round_away(x: np.float32) -> int:
    """Int64(x.rounded()) -- .toNearestOrAwayFromZero; ValueError where Swift traps."""
    if not np.isfinite(x):
        raise ValueError("not finite")
    f = float(x)
    r = math.floor(abs(f) + 0.5) * (1 if f >= 0 else -1)   # exact: |f| < 2^24 has a .5 fraction, larger are integers
    if not -(1 << 63) <= r < 1 << 63:
        raise ValueError("outside Int64")
    return int(r)


def max_scaling_factor(vector_dimension: int, plaintext_moduli) -> int:
    """ClientConfig.maxScalingFactor (Config.swift:112-120) for cosine similarity."""
    t = F32(1)
    for m in plaintext_moduli:
        t = F32(t * float32_of_int(m))
    value = F32(F32(np.sqrt(F32(F32(t - F32(1)) / F32(2)))) - F32(F32(np.sqrt(float32_of_int(vector_dimension))) / F32(2)))
    return int(math.floor(float(value)))


def crt_compose(residues, moduli) -> list:
    """CrtComposer.compose (CrtComposer.swift:76-97): residues[i][j] mod moduli[i] -> values in [0, prod)."""
    q = math.prod(int(m) for m in moduli)
    out = [0] * len(residues[0])
    for m, row in zip(moduli, residues):
        m = int(m)
        inv = pow(q // m, -1, m)
        for j, x in enumerate(row):
            out[j] = (out[j] + (int(x) * inv % m) * (q // m)) % q
    return out


def remainder_to_centered(x: int, modulus: int) -> int:
    return x - modulus if x > (modulus - 1) >> 1 else x


def fixed_point_cosine_similarity(lhs, rhs, modulus: int, scaling_factor) -> np.ndarray:
    """Array2d.fixedPointCosineSimilarity (Util.swift:141-152): lhs rows x d, rhs d x q (its columns normalised);
    the centred modular product (:99-123) over Float(s) * Float(s)."""
    a = normalized_scaled_and_rounded(lhs, scaling_factor)
    b = normalized_scaled_and_rounded(np.asarray(rhs, dtype=np.float32).T.tolist(), scaling_factor)
    return distances_from_signed(mul_mod(a, [list(c) for c in zip(*b)], modulus), scaling_factor)


def mul_mod(x, y, modulus: int) -> list:
    """Array2d<SignedScalar>.mul(_:modulus:) (Util.swift:99-123): the product mod `modulus`, each value centred."""
    return [[remainder_to_centered(sum(int(p) * int(q) for p, q in zip(row, col)) % modulus, modulus) for col in zip(*y)]
            for row in x]


def distances_from_signed(values, scaling_factor) -> np.ndarray:
    """Float(signed) / (Float(s) * Float(s)) (Client.swift:114-117)."""
    s = F32(scaling_factor)
    denom = F32(s * s)
    return np.array([[F32(float32_of_int(v) / denom) for v in row] for row in values], dtype=np.float32)


def generate_query(ctxs: list, sk, vectors, scaling_factor, a_seeds, e_seeds) -> list:
    """Client.generateQuery (Client.swift:73-91): per context the .denseRow plaintexts of the normalised values, each
    encrypted with client_oracle.encrypt under its seeds (a_seeds[k][i], e_seeds[k][i]).  Raises ValueError for a
    value outside the centred range when there is one context."""
    values = normalized_scaled_and_rounded(vectors, scaling_factor)
    rows, cols = len(values), len(values[0])
    flat = [v for row in values for v in row]
    out = []
    for k, ctx in enumerate(ctxs):
        if len(ctxs) == 1 and any(v > (ctx.t - 1) // 2 or v < -(ctx.t // 2) for v in flat):
            raise ValueError("centeredToRemainder: value outside the centred range")
        plain = opn.dense_row_plaintexts(ctx, rows, cols, flat)
        out.append(np.stack([co.encrypt(ctx.n, ctx.q[:ctx.L], ctx.t, sk, p, a_seeds[k][i], e_seeds[k][i])
                             for i, p in enumerate(plain)]))
    return out


def decrypt_values(ctxs: list, sk, replies: list, row_count: int, column_count: int) -> list:
    """Client.decrypt up to the integers (Client.swift:99-117): decrypt, decode and unpack each context's .denseColumn
    replies, CRT-compose, centre over prod t.  Returns row_count x column_count signed values."""
    moduli = [ctx.t for ctx in ctxs]
    unpacked = [opn.unpack_dense_column(ctx, [opn.decode_simd(ctx, ctx.decrypt(sk, ct)).tolist() for ct in cts], row_count, column_count)
                for ctx, cts in zip(ctxs, replies)]
    composed = crt_compose(unpacked, moduli)
    t = math.prod(moduli)
    flat = [remainder_to_centered(v, t) for v in composed]
    return [flat[r * column_count:(r + 1) * column_count] for r in range(row_count)]


def decrypt(ctxs: list, sk, replies: list, row_count: int, column_count: int, scaling_factor) -> np.ndarray:
    """Client.decrypt (Client.swift:99-127): float32 distances, row_count x column_count."""
    return distances_from_signed(decrypt_values(ctxs, sk, replies, row_count, column_count), scaling_factor)


def database_for_testing(row_count: int, vector_dimension: int, metadata_count: int = 0) -> list:
    """PrivateNearestNeighborSearchUtil.getDatabaseForTesting (PnnsUtils.swift:37-45): (entryId, metadata, vector) rows,
    vector[j] = Float(j + row) * (row even ? 1 : -1)."""
    return [(r, bytes([r % 255] * metadata_count), [float(j + r) * (1 if r % 2 == 0 else -1) for j in range(vector_dimension)])
            for r in range(row_count)]


def normalized_scaled_and_rounded_array(vectors, scaling_factor) -> np.ndarray:
    """normalized_scaled_and_rounded over a float32 rows x cols array, vectorised across rows: the same float32 steps
    (the column loop keeps each row's sum left to right).  Raises ValueError where Swift traps."""
    v = np.ascontiguousarray(np.asarray(vectors, dtype=np.float32))
    if not np.all(np.isfinite(v)):
        raise ValueError("not finite")
    s = F32(scaling_factor)
    with np.errstate(all="ignore"):
        total = np.zeros(v.shape[0], dtype=np.float32)
        for k in range(v.shape[1]):
            total = (total + v[:, k] * v[:, k]).astype(np.float32)
        norm = np.sqrt(total).astype(np.float32)
        q = ((v * s).astype(np.float32) / np.where(norm == 0, F32(1), norm)[:, None]).astype(np.float32)
    if not np.all(np.isfinite(q)):
        raise ValueError("not finite")
    d = q.astype(np.float64)
    r = np.floor(np.abs(d) + 0.5) * np.sign(d)          # .toNearestOrAwayFromZero, exact in double
    if np.any(np.abs(r) >= 2.0 ** 63):
        raise ValueError("outside Int64")
    r = r.astype(np.int64)
    r[norm == 0] = 0
    return r
