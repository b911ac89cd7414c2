"""The SimplePIR client's seeded precompute restated in Python integers, the checker of hecuda.simple_pir's device
client (csrc/simple_pir_client.cu):

    generateSecretPolys over NistAes128Ctr(secret seed)      SimplePir+Client.swift:20-28, PolyRq+Randomize.swift:87-104
    noiselessSample, divideAndRound, encryptZero             SimplePir+Client.swift:29-82, Array2d.swift:382-429, 489-514
    add(index:)                                              SimplePir+Precompute.swift:241-256
    resultsWithoutResponse = multiply(transposing:modulus:)  SimplePir+Precompute.swift:122-188

Secret i, coefficient j is stream coefficient i N + j of one ternary stream; error (i, c) is stream coefficient i K + c
of one CBD stream.  The results are computed the reference's way: the secrets mod p, the sum of products taken mod
2^(2 word_bits) (its T.DoubleWidth with &+=), then mod p; `exact` skips the wrap.
"""
from __future__ import annotations

import numpy as np

from oracle import client_oracle as cl
from oracle import simple_pir_oracle as osp


def secrets_from_seed(seed: bytes, cpe: int, n: int) -> np.ndarray:
    return np.array(cl.ternary_values(seed, cpe * n), dtype=np.int64).reshape(cpe, n)


def errors_from_seed(seed: bytes, cpe: int, k: int, std_dev: float) -> np.ndarray:
    return np.array(cl.cbd_values(seed, cpe * k, std_dev), dtype=np.int64).reshape(cpe, k)


def exact_products(secrets_: np.ndarray, hint: np.ndarray):
    """(P, Nn): hint . [s = 1] and hint . [s = -1] per secret row, as Python ints (cpe x M)."""
    h = np.asarray(hint, dtype=np.uint64)
    pos = (secrets_ == 1).astype(np.int64)
    neg = (secrets_ == -1).astype(np.int64)
    out = []
    for mask in (pos, neg):
        acc = np.zeros((secrets_.shape[0], h.shape[0]), dtype=object)
        for shift in range(0, 64, 16):
            limb = ((h >> np.uint64(shift)) & np.uint64(0xFFFF)).astype(np.int64)
            acc = acc + (mask @ limb.T).astype(object) * (1 << shift)
        out.append(acc)
    return out


def results(secrets_: np.ndarray, hint: np.ndarray, p: int, word_bits: int, exact: bool = False) -> np.ndarray:
    pos, neg = exact_products(secrets_, hint)
    u = pos + (p - 1) * neg
    if not exact:
        u = u % (1 << (2 * word_bits))
    return (u % p).astype(np.uint64)


def precompute(prm: dict, hint: np.ndarray, a_seed: bytes, secret_seed: bytes, error_seed: bytes, index=None,
               word_bits: int = 64, std_dev: float = 6.4, exact: bool = False):
    """One query -> (queries cpe x K, results cpe x M, signed secrets cpe x N).  prm: N, pt, ct, entries_per_column,
    chunks_per_entry, database_columns."""
    n, pt, ct = prm["N"], prm["pt"], prm["ct"]
    cpe, epc, k = prm["chunks_per_entry"], prm["entries_per_column"], prm["database_columns"]
    p = osp.ntt_friendly_mod(ct, n)
    polys = osp.a_polynomials(a_seed, n, -(-k // n), p)
    s = secrets_from_seed(secret_seed, cpe, n)
    sample = osp.noiseless_sample(s, osp.a_matrix(polys, k, p), p)
    mask = (1 << ct) - 1
    q = osp.mod_switch(sample, p, ct).astype(object)
    q = (q + (errors_from_seed(error_seed, cpe, k, std_dev).astype(object) % (1 << ct))) & mask
    if index is not None:
        for i in range(cpe):
            col = (index * cpe + i) // epc
            q[i, col] = (q[i, col] + (1 << (ct - pt))) & mask
    return q.astype(np.uint64), results(s, hint, p, word_bits, exact), s
