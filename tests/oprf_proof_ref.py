"""Restatement of the reference's OprfServer.computeResponse (SymmetricPir/SymmetricPirProtocol.swift:39-59) and of its
OprfClient, for the tests, on top of oracle/oprf_oracle.py (P-384, RFC 9380 hashing, RFC 9497 Evaluate/Blind/Finalize).

swift-crypto's P384._VOPRF.PrivateKey.evaluate is RFC 9497 BlindEvaluate (3.3.2) with GenerateProof (2.2.1) over one
element, returned as SerializeElement(k B) || SerializeScalar(c) || SerializeScalar(s).  The proof nonce r is drawn as
proof_nonce describes; a verifier accepts any r in [1, n - 1].  Like CONTEXT_STRING, the proof's bytes follow RFC 9497's
text: no swift-crypto vector on hand pins them.
"""
from __future__ import annotations

import hashlib
from typing import List, Optional, Sequence, Tuple

from oracle.oprf_oracle import (AES_KEY_BYTES, CONTEXT_STRING, ELEMENT_BYTES, KEY_BYTES, KEYWORD_BYTES, NONCE_BYTES, G,
                                N, Point, add, blind, check_key, deserialize_element, expand_message_xmd, finalize,
                                hash_to_group, i2osp, mul, serialize_element)
HASH_TO_SCALAR_DST = b"HashToScalar-" + CONTEXT_STRING
SEED_DST = b"Seed-" + CONTEXT_STRING
PROOF_NONCE_DST = b"HECUDA-ProofNonce-" + CONTEXT_STRING
SCALAR_BYTES, PROOF_BYTES, RESPONSE_BYTES, NONCE_SEED_BYTES = 48, 96, 145, 32


def hash_to_scalar(msg: bytes) -> int:
    """RFC 9380 hash_to_field with modulus n, L = 72, count 1, DST "HashToScalar-" || contextString."""
    return int.from_bytes(expand_message_xmd(msg, HASH_TO_SCALAR_DST, 72), "big") % N


def serialize_scalar(s: int) -> bytes:
    return i2osp(s % N, SCALAR_BYTES)


def _framed(data: bytes) -> bytes:
    return i2osp(len(data), 2) + data


def _composite_weights(pkS: Point, Cs: Sequence[Point], Ds: Sequence[Point]) -> List[int]:
    seed = hashlib.sha384(_framed(serialize_element(pkS)) + _framed(SEED_DST)).digest()
    return [hash_to_scalar(_framed(seed) + i2osp(i, 2) + _framed(serialize_element(c)) + _framed(serialize_element(d)) +
                           b"Composite") for i, (c, d) in enumerate(zip(Cs, Ds))]


def compute_composites_fast(k: int, pkS: Point, Cs: Sequence[Point], Ds: Sequence[Point]) -> Tuple[Point, Point]:
    """ComputeCompositesFast (2.2.1): M = sum d_i C_i, Z = k M."""
    M: Point = None
    for d, c in zip(_composite_weights(pkS, Cs, Ds), Cs):
        M = add(M, mul(d, c))
    return M, mul(k, M)


def compute_composites(pkS: Point, Cs: Sequence[Point], Ds: Sequence[Point]) -> Tuple[Point, Point]:
    """ComputeComposites (2.2.2, the verifier's): M = sum d_i C_i, Z = sum d_i D_i."""
    M: Point = None
    Z: Point = None
    for d, c, e in zip(_composite_weights(pkS, Cs, Ds), Cs, Ds):
        M, Z = add(M, mul(d, c)), add(Z, mul(d, e))
    return M, Z


def _challenge(pkS: Point, M: Point, Z: Point, t2: Point, t3: Point) -> int:
    return hash_to_scalar(b"".join(_framed(serialize_element(p)) for p in (pkS, M, Z, t2, t3)) + b"Challenge")


def generate_proof(k: int, r: int, B: Point, D: Point) -> bytes:
    """GenerateProof(k, G, k G, [B], [D]) with nonce r: SerializeScalar(c) || SerializeScalar(s)."""
    pkS = mul(k, G)
    M, Z = compute_composites_fast(k, pkS, [B], [D])
    c = _challenge(pkS, M, Z, mul(r, G), mul(r, M))
    return serialize_scalar(c) + serialize_scalar(r - c * k)


def verify_proof(pkS: Point, B: Point, D: Point, proof: bytes) -> bool:
    """VerifyProof(G, pkS, [B], [D], proof) (2.2.2)."""
    if len(proof) != PROOF_BYTES:
        return False
    c, s = int.from_bytes(proof[:SCALAR_BYTES], "big"), int.from_bytes(proof[SCALAR_BYTES:], "big")
    if c >= N or s >= N:
        return False
    M, Z = compute_composites(pkS, [B], [D])
    t2 = add(mul(s, G), mul(c, pkS))
    t3 = add(mul(s, M), mul(c, Z))
    return _challenge(pkS, M, Z, t2, t3) == c


def proof_nonce(k: int, seed: bytes, blinded: bytes) -> int:
    """r = OS2IP(expand_message_xmd(I2OSP(k, 48) || seed || Ser(B), "HECUDA-ProofNonce-" || contextString, 72)) mod n."""
    assert len(seed) == NONCE_SEED_BYTES
    return int.from_bytes(expand_message_xmd(i2osp(k, KEY_BYTES) + seed + blinded, PROOF_NONCE_DST, 72), "big") % N


def blind_evaluate_verifiable(secret_key: bytes, query: bytes, seed: bytes) -> bytes:
    """BlindEvaluate with the proof: 145 bytes.  ValueError for an invalid query (or r = 0)."""
    k = check_key(secret_key)
    B = deserialize_element(bytes(query))
    D = mul(k, B)
    r = proof_nonce(k, seed, serialize_element(B))
    if r == 0:
        raise ValueError("proof nonce is 0")
    return serialize_element(D) + generate_proof(k, r, B, D)


def finalize_verifiable(data: bytes, blind_scalar: int, response: bytes, pkS: bytes) -> bytes:
    """Finalize (3.3.2) of one input: verify the proof against the blinded element r HashToGroup(data), then unblind and
    hash.  ValueError when the proof does not verify."""
    if len(response) != RESPONSE_BYTES:
        raise ValueError("response length")
    B = mul(blind_scalar, hash_to_group(data))
    D = deserialize_element(response[:ELEMENT_BYTES])
    if not verify_proof(deserialize_element(pkS), B, D, response[ELEMENT_BYTES:]):
        raise ValueError("VerifyError")
    return finalize(data, blind_scalar, response[:ELEMENT_BYTES])


class OprfClient:
    """OprfClient (SymmetricPir/SymmetricPirProtocol.swift:62-134): queryContext -> (blind, keyword, query), parse
    verifies, finalizes and splits the output into (obliviousKeyword, nonce, secretKey), decrypt opens an entry."""

    def __init__(self, serverPublicKey: bytes):
        deserialize_element(serverPublicKey)
        self.serverPublicKey = bytes(serverPublicKey)

    def queryContext(self, keyword: bytes, blind_scalar: Optional[int] = None) -> Tuple[int, bytes, bytes]:
        r, query = blind(bytes(keyword), blind_scalar)
        return r, bytes(keyword), query

    def parse(self, response: bytes, context: Tuple[int, bytes, bytes]) -> Tuple[bytes, bytes, bytes]:
        r, keyword, _ = context
        h = finalize_verifiable(keyword, r, bytes(response), self.serverPublicKey)
        return h[:KEYWORD_BYTES], h[:NONCE_BYTES], h[-AES_KEY_BYTES:]

    @staticmethod
    def decrypt(encryptedEntry: bytes, parsed: Tuple[bytes, bytes, bytes]) -> bytes:
        from cryptography.hazmat.primitives.ciphers.aead import AESGCM

        _, nonce, key = parsed
        return AESGCM(key).decrypt(nonce, bytes(encryptedEntry), None)
