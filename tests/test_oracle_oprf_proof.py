"""Pins tests/oprf_proof_ref.py, the restatement of the OPRF server's BlindEvaluate with the DLEQ proof (RFC 9497 3.3.2,
2.2.1-2.2.2) that the device code is checked against: proofs verify and tampered ones do not, both composites agree,
the verifiable Finalize of a blinded evaluation equals the already pinned Evaluate, r G matches cryptography, and
invalid encodings are rejected."""
import random

import pytest

import oprf_proof_ref as R
from oracle import oprf_oracle as O


def keys(count, seed):
    rng = random.Random(seed)
    return [rng.randrange(1, O.N) for _ in range(count)]


@pytest.mark.parametrize("k", keys(3, 40) + [1, O.N - 1])
def test_proofs_verify_and_tampering_fails(k):
    rng = random.Random(k % 1000)
    B = O.hash_to_group(rng.randbytes(20))
    D = O.mul(k, B)
    pkS = O.mul(k, O.G)
    proof = R.generate_proof(k, rng.randrange(1, O.N), B, D)
    assert R.verify_proof(pkS, B, D, proof)
    c, s = proof[:48], proof[48:]
    flip = (int.from_bytes(c, "big") ^ 1).to_bytes(48, "big")
    assert not R.verify_proof(pkS, B, D, flip + s)
    assert not R.verify_proof(pkS, B, D, c + ((int.from_bytes(s, "big") + 1) % O.N).to_bytes(48, "big"))
    assert not R.verify_proof(pkS, B, O.add(D, O.G), proof)
    assert not R.verify_proof(O.mul(k % (O.N - 1) + 1, O.G), B, D, proof)


def test_composites_agree():
    for k in keys(3, 41):
        B = O.hash_to_group(b"composite %d" % k)
        D = O.mul(k, B)
        pkS = O.mul(k, O.G)
        assert R.compute_composites_fast(k, pkS, [B], [D]) == R.compute_composites(pkS, [B], [D])


def test_finalize_of_the_blind_path_is_evaluate():
    rng = random.Random(42)
    for k in keys(3, 43):
        key = k.to_bytes(48, "big")
        pk = O.public_key(key)
        for _ in range(2):
            data = rng.randbytes(rng.randrange(0, 60))
            blind_scalar, query = O.blind(data, rng.randrange(1, O.N))
            response = R.blind_evaluate_verifiable(key, query, rng.randbytes(32))
            assert len(response) == 145
            assert R.finalize_verifiable(data, blind_scalar, response, pk) == O.evaluate(key, data)


def test_nonce_is_deterministic_and_hedged():
    key, query = (5).to_bytes(48, "big"), O.blind(b"n", 9)[1]
    assert R.blind_evaluate_verifiable(key, query, bytes(32)) == R.blind_evaluate_verifiable(key, query, bytes(32))
    a, b = R.blind_evaluate_verifiable(key, query, bytes(32)), R.blind_evaluate_verifiable(key, query, b"\1" * 32)
    assert a[:49] == b[:49] and a[49:] != b[49:]


def test_client_round_trip():
    key = keys(1, 44)[0].to_bytes(48, "big")
    client = R.OprfClient(O.public_key(key))
    context = client.queryContext(b"keyword")
    parsed = client.parse(R.blind_evaluate_verifiable(key, context[2], bytes(32)), context)
    h = O.evaluate(key, b"keyword")
    assert parsed == (h[:16], h[:12], h[24:])
    assert client.decrypt(O.seal(h, b"value"), parsed) == b"value"


@pytest.mark.parametrize("r", [1, 2, 3, O.N - 1] + keys(3, 45))
def test_r_g_matches_cryptography(r):
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric import ec

    expected = ec.derive_private_key(r, ec.SECP384R1()).public_key().public_bytes(
        serialization.Encoding.X962, serialization.PublicFormat.CompressedPoint)
    assert O.serialize_element(O.mul(r, O.G)) == expected


def invalid_encodings():
    good = O.blind(b"x", 7)[1]
    off_curve = next(x for x in range(1, 100) if not O.is_square((x ** 3 + O.A * x + O.B) % O.P))
    return {"prefix 0": b"\0" + good[1:], "prefix 1": b"\1" + good[1:], "prefix 4": b"\4" + good[1:],
            "x = p": b"\2" + O.P.to_bytes(48, "big"), "x > p": b"\3" + (O.P + 5).to_bytes(48, "big"),
            "off curve": b"\2" + off_curve.to_bytes(48, "big"), "zeros": bytes(49)}


@pytest.mark.parametrize("name", sorted(invalid_encodings()))
def test_invalid_encodings_are_rejected(name):
    with pytest.raises(ValueError):
        R.blind_evaluate_verifiable((3).to_bytes(48, "big"), invalid_encodings()[name], bytes(32))
