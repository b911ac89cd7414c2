"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's BFV client: key generation, symmetric encryption,
key-switching keys and the noise budget, with every random polynomial drawn from a NistAes128Ctr stream (drbg_oracle).

Only tests/ and tools/ may import this module; the product (swift-homomorphic-encryption_b200/) never does.

  * ternary map      PolyRq.randomizeTernary(using:)          PolyRq/PolyRq+Randomize.swift:87-104
  * CBD map          randomizeCenteredBinomialDistribution     PolyRq/PolyRq+Randomize.swift:120-160
  * rng.next() -> T  sizeof(T) bytes, little-endian           Random/PseudoRandomNumberGenerator.swift:37-43
  * secret key       Bfv.generateSecretKey                     Bfv/Bfv+Keys.swift:20-26
  * encryption       Bfv.encrypt / encryptZero                 Bfv/Bfv+Encrypt.swift:64-181 (plaintextTranslate :75-139)
  * key switching    _generateKeySwitchKey, generateEvaluationKey  Bfv/Bfv+Keys.swift:30-103
  * noise budget     Bfv.noiseBudgetEval / noiseBudgetCoeff    Bfv/Bfv+Decrypt.swift:116-185

The reference draws the secret and the error from SystemRandomNumberGenerator; here, as in the device code, each has its
own seeded stream, and the maps from stream bytes to coefficients are the reference's.  Arithmetic is on Python
integers; the NTTs are the C oracle's (oracle.py).
"""
from __future__ import annotations

import math

import numpy as np

from . import oracle as O
from .drbg_oracle import NistAes128Ctr, random_poly

STD_DEV_32, STD_DEV_64 = 3.2, 6.4  # ErrorStdDev.stdDev32 / stdDev64 (EncryptionParameters.swift:32-38)


def _residues(values, moduli) -> np.ndarray:
    """Small signed integers per coefficient -> (rows, N) residues, value mod q_i on every row."""
    return np.array([[v % int(q) for v in values] for q in moduli], dtype=np.uint64)


def ternary_values(seed: bytes, n: int) -> list:
    """randomizeTernary: coefficient j = ((UInt64 << 32 | UInt32) mod 3) - 1, 12 stream bytes per coefficient."""
    data = NistAes128Ctr(seed).fill(12 * n)
    out = []
    for j in range(n):
        hi = int.from_bytes(data[12 * j:12 * j + 8], "little")
        lo = int.from_bytes(data[12 * j + 8:12 * j + 12], "little")
        out.append(((hi << 32) | lo) % 3 - 1)
    return out


def cbd_shape(std_dev: float):
    """(k, UInt64 words per coefficient, mask of the last word of each half) for a standard deviation."""
    k = math.ceil(2 * std_dev * std_dev)  # Int((2 * variance).rounded(.up))
    words = 2 * -(-k // 64)
    mask = (1 << (k % 64)) - 1 if k % 64 else (1 << 64) - 1
    return k, words, mask


def cbd_values(seed: bytes, n: int, std_dev: float = STD_DEV_32) -> list:
    """randomizeCenteredBinomialDistribution: popcount of the first half of the trial words minus the second half's."""
    _, words, mask = cbd_shape(std_dev)
    half = words // 2
    data = NistAes128Ctr(seed).fill(8 * words * n)
    out = []
    for j in range(n):
        trial = [int.from_bytes(data[8 * (j * words + w):8 * (j * words + w + 1)], "little") for w in range(words)]
        trial[half - 1] &= mask
        trial[words - 1] &= mask
        out.append(sum(x.bit_count() for x in trial[:half]) - sum(x.bit_count() for x in trial[half:]))
    return out


def generate_secret_key(n: int, moduli, seed: bytes) -> np.ndarray:
    """Bfv.generateSecretKey over every coefficient modulus (secretKeyContext) -> (K, N) Eval."""
    return O.ntt_forward(n, moduli, _residues(ternary_values(seed, n), moduli))


def _mul(a, b, moduli) -> np.ndarray:
    q = np.array([int(m) for m in moduli], dtype=object)[:, None]
    return ((np.asarray(a).astype(object) * np.asarray(b).astype(object)) % q).astype(np.uint64)


def _add(a, b, moduli) -> np.ndarray:
    q = np.array([int(m) for m in moduli], dtype=object)[:, None]
    return ((np.asarray(a).astype(object) + np.asarray(b).astype(object)) % q).astype(np.uint64)


def _neg(a, moduli) -> np.ndarray:
    q = np.array([int(m) for m in moduli], dtype=object)[:, None]
    return ((-np.asarray(a).astype(object)) % q).astype(np.uint64)


def encrypt_zero(n: int, moduli, sk, a_seed: bytes, e_seed: bytes, std_dev: float = STD_DEV_32) -> np.ndarray:
    """encryptZero over `moduli` (Bfv+Encrypt.swift:150-181) -> (2, rows, N) Coeff: (-(INTT(a s) + e), INTT(a))."""
    rows = len(moduli)
    a = random_poly(n, moduli, a_seed)                    # sampled in Eval
    e = _residues(cbd_values(e_seed, n, std_dev), moduli)
    c0 = _add(O.ntt_inverse(n, moduli, _mul(a, np.asarray(sk)[:rows], moduli)), e, moduli)
    return np.stack([_neg(c0, moduli), O.ntt_inverse(n, moduli, a)])


def translate_add(n: int, moduli, t: int, ct, plain) -> np.ndarray:
    """plaintextTranslate(.Add) (Bfv+Encrypt.swift:75-139): c0 += floor(Q/t) m + floor(([Q]_t m + (t+1)/2) / t)."""
    q_prod = math.prod(int(q) for q in moduli)
    out = np.array(ct, dtype=np.uint64, copy=True)
    threshold = (t + 1) // 2
    for j in range(n):
        m = int(plain[j])
        adjust = ((q_prod % t) * m + threshold) // t
        for i, q in enumerate(moduli):
            q = int(q)
            out[0, i, j] = (int(out[0, i, j]) + ((q_prod // t) % q * m + adjust)) % q
    return out


def encrypt(n: int, moduli, t: int, sk, plain, a_seed: bytes, e_seed: bytes) -> np.ndarray:
    """Bfv.encrypt at the ciphertext level `moduli` -> (2, L, N) Coeff."""
    return translate_add(n, moduli, t, encrypt_zero(n, moduli, sk, a_seed, e_seed), plain)


def key_switch_key(n: int, ct_moduli, q_ks: int, current_key, sk, a_seeds, e_seeds, rows=None) -> np.ndarray:
    """_generateKeySwitchKey (Bfv+Keys.swift:67-103) -> (L, 2, K, N) Eval: key ciphertext i = forwardNtt(encryptZero over
    [q_0..q_{L-1}, q_ks]) with (q_ks mod q_i) currentKey[i] added to row i of poly0.  rows: only the key ciphertexts i
    in `rows`, in that order ((len(rows), 2, K, N)); each has its own seeds, so they equal those of the whole key."""
    ks = [int(q) for q in ct_moduli] + [int(q_ks)]
    out = []
    for i in (range(len(ct_moduli)) if rows is None else rows):
        ct = encrypt_zero(n, ks, sk, a_seeds[i], e_seeds[i])
        ev = np.stack([O.ntt_forward(n, ks, ct[p]) for p in range(2)])
        q = int(ct_moduli[i])
        ev[0, i] = (ev[0, i].astype(object) + (int(q_ks) % q) * np.asarray(current_key)[i].astype(object)) % q
        out.append(ev)
    return np.stack(out)


def generate_evaluation_key(n: int, ct_moduli, q_ks: int, sk, has_relin: bool, elements, a_seeds, e_seeds, rows=None):
    """Bfv.generateEvaluationKey (Bfv+Keys.swift:30-65) with seeds in hecuda_evk_generate's order (the relinearization
    key, then the elements, L per key) -> (relinearization key or None, {element: key}); rows as in key_switch_key."""
    L = len(ct_moduli)
    ks = [int(q) for q in ct_moduli] + [int(q_ks)]
    sk = np.asarray(sk)
    keys, used = [], 0
    currents = ([_mul(sk, sk, ks)] if has_relin else []) + [O.galois_eval(n, L + 1, g, sk) for g in elements]
    for current in currents:
        keys.append(key_switch_key(n, ct_moduli, q_ks, current, sk, a_seeds[used:used + L], e_seeds[used:used + L], rows))
        used += L
    relin = keys.pop(0) if has_relin else None
    return relin, dict(zip(elements, keys))


def noise_norm(n: int, moduli, t: int, sk, ct, eval_format: bool = False) -> int:
    """The infinity norm of [t (c0 + c1 s (+ c2 s^2))]_q, centred, as noiseBudgetEval computes it."""
    ct = np.asarray(ct)
    polys, l = ct.shape[0], ct.shape[1]
    q = [int(m) for m in moduli[:l]]
    ev = ct if eval_format else np.stack([O.ntt_forward(n, q, ct[p]) for p in range(polys)])
    s = np.asarray(sk)[:l]
    dot, power = ev[0], s
    for k in range(1, polys):
        dot = _add(dot, _mul(ev[k], power, q), q)
        power = _mul(power, s, q)
    v = O.ntt_inverse(n, q, dot)
    q_prod = math.prod(q)
    half = (q_prod + 1) >> 1
    weights = [(q_prod // qi) * pow(q_prod // qi, -1, qi) for qi in q]
    norm = 0
    for j in range(n):
        coeff = sum(int(v[i, j]) * t * w for i, w in enumerate(weights)) % q_prod
        norm = max(norm, q_prod - coeff if coeff > half else coeff)
    return norm


def noise_budget(n: int, moduli, t: int, sk, ct, eval_format: bool = False) -> float:
    """Bfv.noiseBudgetEval / noiseBudgetCoeff: log2(qDouble / (2 norm)), inf for a zero norm."""
    norm = noise_norm(n, moduli, t, sk, ct, eval_format)
    if norm == 0:
        return math.inf
    q_double = 1.0
    for qi in moduli[:np.asarray(ct).shape[1]]:
        q_double *= float(int(qi))
    return math.log2(q_double / (2 * float(norm)))
