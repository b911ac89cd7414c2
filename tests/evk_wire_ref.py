"""TEST INFRASTRUCTURE ONLY -- seeded evaluation keys for the wire-format key tests (tests/test_*_evk_wire.py).

  * EvaluationKey(deserialize:) of a .seeded key-switching ciphertext (SerializedKeys.swift:141-157,
    SerializedCiphertext.swift:41-60 with Format = Eval): poly0 = PolyRq(deserialize:) over the key-switching rows
    [q_0..q_{L-1}, q_ks], poly1 = PolyRq.random over the same rows from NistAes128Ctr(seed:).  Keys are Eval and `a` is
    sampled in Eval (Bfv+Encrypt.swift:156-157), so there is no NTT.
  * reseed_key: an oracle key-switching key re-expressed with DRBG-sampled `a`, as _generateKeySwitchKey produces it
    (encryptZero keeps its seed, Bfv+Encrypt.swift:150-181): c0' = c0 + (a - a_seed) s, a' = a_seed.  c0' + a' s is
    unchanged, so the key carries the same error and switches the same way.
  * reseed_query: the same trick for a Coeff query ciphertext (the c1 of SerializedCiphertext.seeded is the seed's
    random Eval polynomial converted to Coeff).

Built from oracle.drbg_oracle.random_poly and oracle.pir_oracle's codec, both pinned against the reference.
"""
import numpy as np

from oracle import drbg_oracle as drbg
from oracle import oracle as orc
from oracle import pir_oracle as opir


def expand_seeded_key_ciphertext(ctx, poly0: bytes, seed: bytes) -> np.ndarray:
    """One seeded key-switching ciphertext -> (2, K, N) Eval over [q_0..q_{L-1}, q_ks]."""
    moduli = ctx.moduli
    return np.stack([opir.load_poly(ctx.n, moduli, poly0), drbg.random_poly(ctx.n, moduli, seed)])


def reseed_key(ctx, sk, key, seeds):
    """key (L, 2, K, N) Eval and the secret key sk (K, N) Eval -> (the seeded key (L, 2, K, N), poly0 bytes (L, B))."""
    n, moduli = ctx.n, ctx.moduli
    s = np.asarray(sk, dtype=np.uint64)
    out, wire = np.array(key, dtype=np.uint64, copy=True), []
    for i, seed in enumerate(seeds):
        a_seed = drbg.random_poly(n, moduli, bytes(seed))
        delta = orc.poly_op("sub", n, moduli, out[i, 1], a_seed)
        out[i, 0] = orc.poly_op("add", n, moduli, out[i, 0], orc.poly_op("mul", n, moduli, delta, s))
        out[i, 1] = a_seed
        wire.append(np.frombuffer(opir.serialize_poly(n, moduli, out[i, 0]), dtype=np.uint8))
    return out, np.stack(wire)


def reseed_query(ctx, sk, query, seeds):
    """Coeff query ciphertexts (count, 2, L, N) -> (the seeded ciphertexts, poly0 bytes (count, byteCount(L rows)))."""
    n, q = ctx.n, ctx.q
    s_eval = np.asarray(sk, dtype=np.uint64)[: ctx.L]
    cts, wire = [], []
    for ct, seed in zip(query, seeds):
        a_eval = drbg.random_poly(n, q, bytes(seed))
        delta = orc.poly_op("sub", n, q, orc.ntt_forward(n, q, ct[1]), a_eval)
        c0 = orc.poly_op("add", n, q, ct[0], orc.ntt_inverse(n, q, orc.poly_op("mul", n, q, delta, s_eval)))
        cts.append(np.stack([c0, orc.ntt_inverse(n, q, a_eval)]))
        wire.append(np.frombuffer(opir.serialize_poly(n, q, c0), dtype=np.uint8))
    return np.stack(cts), np.stack(wire)


def random_seeds(rng, count):
    return rng.integers(0, 256, size=(count, 32), dtype=np.uint8)
