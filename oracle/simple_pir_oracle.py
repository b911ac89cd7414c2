"""SimplePIR server semantics restated in Python integers (Sources/PrivateInformationRetrieval/SimplePir/), the checker of
hecuda.simple_pir:

    computingParams                       SimplePir+Database.swift:208-243
    process (A materialised, dense DB'.A) SimplePir+Database.swift:177-206, 252-290
    computeResponse                       SimplePir+Server.swift:31-38, Array2d.multiply(transposing:mask:)
    extractEntries / noiseless decode     SimplePir+Client.swift:85-95, SimplePir+Precompute.swift:284-296
    the client: secret keys, noiselessSample, encryptZero with modSwitch, add(index:), integrate and decrypt
                                          SimplePir+Client.swift, SimplePir+Precompute.swift:199-312
"""
from __future__ import annotations

import math

import numpy as np

from oracle import oracle as O
from oracle.drbg_oracle import NistAes128Ctr
from oracle.pir_oracle import bytes_to_coefficients, coefficients_to_bytes


def coeff_count(byte_count: int, bits: int) -> int:
    return -(-8 * byte_count // bits)


def swift_rounded(x: float) -> int:  # Double.rounded(): halves away from zero (x >= 0 here)
    return math.floor(x + 0.5)


def computing_params(pt: int, entry_count: int, entry_size: int) -> dict:
    scalars = coeff_count(entry_size, pt)
    ideal = min(swift_rounded(math.sqrt(float(entry_count * scalars))), scalars)
    epc = max(swift_rounded(float(ideal) / float(scalars)), 1)
    cpe = max(int(float(scalars) / float(ideal)), 1)
    columns = entry_count * cpe if epc == 1 else max(-(-entry_count // epc), 1)
    return dict(entry_scalars=scalars, entries_per_column=epc, chunks_per_entry=cpe, database_columns=columns)


def shape(pt: int, entry_size: int, epc: int, cpe: int):
    scalars = coeff_count(entry_size, pt)
    chunk = -(-scalars // cpe)
    column_size = epc * scalars if cpe == 1 else chunk
    padded = scalars if cpe == 1 else -(-scalars // cpe) * cpe
    return scalars, padded, column_size, chunk


def ntt_friendly_mod(ct: int, n: int) -> int:
    return O.generate_primes([ct + 1], True, n)[0]


def process_database(entries: np.ndarray, pt: int, epc: int, cpe: int, columns: int) -> np.ndarray:
    """The processed database DB' (columnSize x databaseColumns) as Python-int-valued uint64."""
    entries = np.asarray(entries, dtype=np.uint8)
    scalars, padded, column_size, _ = shape(pt, entries.shape[1], epc, cpe)
    flat = np.zeros(columns * column_size, dtype=np.uint64)
    for e in range(entries.shape[0]):
        flat[e * padded:e * padded + scalars] = bytes_to_coefficients(entries[e].tobytes(), pt, False)
    return flat.reshape(columns, column_size).T.copy()


def a_polynomials(seed: bytes, n: int, count: int, p: int) -> np.ndarray:
    """generateAPolynomials: `count` PolyRq.random polynomials from one NistAes128Ctr(seed) stream."""
    data = NistAes128Ctr(seed).fill(count * n * 16)
    words = [int.from_bytes(data[16 * i:16 * i + 16], "little") % p for i in range(count * n)]
    return np.array(words, dtype=np.uint64).reshape(count, n)


def a_matrix(polys: np.ndarray, columns: int, p: int) -> np.ndarray:
    """materializeAMatrix: A[jN + k][c] = coef_k(a_j x^c) mod p, truncated to `columns` rows."""
    count, n = polys.shape
    k = np.arange(n)[:, None]
    c = np.arange(n)[None, :]
    src = (k - c) % n
    sign_neg = k < c
    blocks = []
    for j in range(count):
        a = polys[j].astype(np.int64)[src]
        blocks.append(np.where(sign_neg & (a != 0), p - a, a))
    return np.concatenate(blocks, axis=0)[:columns].astype(np.uint64)


def mulmod_matrix(lhs: np.ndarray, rhs: np.ndarray, p: int) -> np.ndarray:
    """(lhs . rhs) mod p exactly, |lhs| < 2^16 (signed allowed), 0 <= rhs < p < 2^62 and inner dimension < 2^31: rhs
    in 15-bit limbs."""
    lhs64 = np.asarray(lhs).astype(np.int64)
    out = np.zeros((lhs.shape[0], rhs.shape[1]), dtype=object)
    r = rhs.astype(np.uint64)
    shift = 0
    while shift < 62:
        limb = ((r >> np.uint64(shift)) & np.uint64(0x7FFF)).astype(np.int64)
        out = out + (lhs64 @ limb).astype(object) * (1 << shift)
        shift += 15
    return (out % p).astype(np.uint64)


def hint(db: np.ndarray, seed: bytes, n: int, p: int) -> np.ndarray:
    columns = db.shape[1]
    polys = a_polynomials(seed, n, -(-columns // n), p)
    return mulmod_matrix(db, a_matrix(polys, columns, p), p)


def negacyclic_mul(a, b, p):
    n = len(a)
    out = [0] * n
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                k = i + j
                if k < n:
                    out[k] = (out[k] + x * y) % p
                else:
                    out[k - n] = (out[k - n] - x * y) % p
    return out


def hint_adjoint(db: np.ndarray, polys: np.ndarray, p: int) -> np.ndarray:
    """hint[r] = coeffs(sum_j sigma(a_j) . d_{r,j}) mod p, sigma(a) = a(x^-1): the identity the device computes."""
    count, n = polys.shape
    out = np.zeros((db.shape[0], n), dtype=np.uint64)
    for r in range(db.shape[0]):
        acc = [0] * n
        for j in range(count):
            a = [int(v) for v in polys[j]]
            sig = [a[0]] + [(-a[n - i]) % p for i in range(1, n)]
            d = [int(v) for v in db[r, j * n:(j + 1) * n]] + [0] * max(0, (j + 1) * n - db.shape[1])
            acc = [(x + y) % p for x, y in zip(acc, negacyclic_mul(sig, d[:n], p))]
        out[r] = acc
    return out


def response(db: np.ndarray, request: np.ndarray, ct: int) -> np.ndarray:
    """computeResponse: transpose((DB' . request^T) mod 2^ct), wrapping products like the reference."""
    prod = np.asarray(db, dtype=np.uint64) @ np.asarray(request, dtype=np.uint64).T  # numpy wraps mod 2^64
    return (prod & np.uint64((1 << ct) - 1)).T.copy()


def selection_request(index: int, pt: int, ct: int, epc: int, cpe: int, columns: int) -> np.ndarray:
    """A noiseless query for entry `index` (PrecomputedQueries.add(index:) on a zero sample): delta at its columns."""
    req = np.zeros((cpe, columns), dtype=np.uint64)
    for q in range(cpe):
        req[q, (index * cpe + q) // epc] = 1 << (ct - pt)
    return req


def decode_noiseless(resp: np.ndarray, index: int, pt: int, ct: int, entry_size: int, epc: int, cpe: int) -> bytes:
    """extractEntries + integrate on a noiseless response, then coefficientsToBytes."""
    scalars, _, column_size, chunk = shape(pt, entry_size, epc, cpe)
    coeffs = []
    for q in range(cpe):
        start = ((index * cpe + q) % epc) * chunk
        row = resp[q, start:start + chunk]
        coeffs += [((int(v) + (1 << (ct - pt - 1))) & ((1 << ct) - 1)) >> (ct - pt) for v in row]
    return coefficients_to_bytes(np.array(coeffs, dtype=np.uint64), pt)[:entry_size]


# ---- the client (SimplePir+Client.swift, SimplePir+Precompute.swift:199-312), for end-to-end tests of the server
def secret_polys(rng, cpe: int, n: int) -> np.ndarray:
    """generateSecretPolys: chunksPerEntry ternary polynomials, as signed values in {-1, 0, 1}."""
    return rng.integers(-1, 2, size=(cpe, n)).astype(np.int64)


def mod_switch(values: np.ndarray, p: int, ct: int) -> np.ndarray:
    """Array2d.divideAndRound(initialMod: p, newMod: 2^ct) (Array2d.swift:489-514): floor((x 2^ct + p / 2) / p) mod 2^ct."""
    return np.array([((int(x) << ct) + (p >> 1)) // p % (1 << ct) for x in np.asarray(values).reshape(-1)],
                    dtype=np.uint64).reshape(np.asarray(values).shape)


def noiseless_sample(secrets_: np.ndarray, a: np.ndarray, p: int) -> np.ndarray:
    """noiselessSample = S . A^T mod p (cpe x K), computed from the materialised A."""
    return mulmod_matrix(secrets_, a.T, p)


def noiseless_sample_polynomial(secrets_: np.ndarray, polys: np.ndarray, columns: int, p: int) -> np.ndarray:
    """noiselessSample as the reference computes it: row i is coeffs(a_j . s_i) for every j, concatenated, cut to K."""
    rows = []
    for s in secrets_:
        sv = [int(v) % p for v in s]
        row = []
        for a in polys:
            row += negacyclic_mul([int(v) for v in a], sv, p)
        rows.append(row[:columns])
    return np.array(rows, dtype=np.uint64)


class Client:
    """SimplePirClient with DefaultQueryGenerator: one precomputed query per call of query(index)."""

    def __init__(self, params: dict, hint: np.ndarray, seed: bytes, rng):
        self.prm, self.rng = params, rng
        self.n, self.pt, self.ct = params["N"], params["pt"], params["ct"]
        self.epc, self.cpe, self.k = params["entries_per_column"], params["chunks_per_entry"], params["database_columns"]
        self.entry_size = params["entry_size"]
        self.p = ntt_friendly_mod(self.ct, self.n)
        self.a = a_matrix(a_polynomials(seed, self.n, -(-self.k // self.n), self.p), self.k, self.p)
        self.hint = np.asarray(hint, dtype=np.uint64)

    def query(self, index: int):
        mask = (1 << self.ct) - 1
        s = secret_polys(self.rng, self.cpe, self.n)
        q = mod_switch(noiseless_sample(s, self.a, self.p), self.p, self.ct)
        # randomCenteredBinomialDistribution(standardDeviation: 6.4): variance 2 x 41 x 1/4 ~ 6.4^2
        err = (self.rng.binomial(82, 0.5, size=q.shape) - 41) % (1 << self.ct)
        q = (q.astype(object) + err.astype(object)) & mask
        delta = 1 << (self.ct - self.pt)
        for qi in range(self.cpe):
            col = (index * self.cpe + qi) // self.epc
            q[qi, col] = (q[qi, col] + delta) & mask
        results = mulmod_matrix(s, self.hint.T, self.p)  # S . hint^T mod p (cpe x M)
        return q.astype(np.uint64), results

    def decrypt(self, response: np.ndarray, results: np.ndarray, index: int) -> bytes:
        mask = (1 << self.ct) - 1
        scalars, _, column_size, chunk = shape(self.pt, self.entry_size, self.epc, self.cpe)
        coeffs = []
        for qi in range(self.cpe):
            start = ((index * self.cpe + qi) % self.epc) * chunk
            for c in range(start, start + chunk):
                v = (int(response[qi, c]) - int(results[qi, c]) + ((1 << (self.ct - self.pt)) >> 1)) & mask
                coeffs.append(v >> (self.ct - self.pt))
        return coefficients_to_bytes(np.array(coeffs, dtype=np.uint64), self.pt)[:self.entry_size]
