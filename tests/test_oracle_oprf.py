"""Pins oracle/oprf_oracle.py, the restatement the symmetric-PIR device code is checked against: the RFC 9380 P-384
vector, scalar multiplication and ECDH against cryptography, the OPRF round trip of the reference's oprfRoundtrip test,
and the sealed rows of its database test."""
import random

import pytest

cryptography = pytest.importorskip("cryptography")
from cryptography.exceptions import InvalidTag  # noqa: E402
from cryptography.hazmat.primitives import serialization  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import ec  # noqa: E402
from cryptography.hazmat.primitives.ciphers.aead import AESGCM  # noqa: E402

from oracle import oprf_oracle as O  # noqa: E402


def compressed_public_key(k: int) -> bytes:
    return ec.derive_private_key(k, ec.SECP384R1()).public_key().public_bytes(serialization.Encoding.X962,
                                                                            serialization.PublicFormat.CompressedPoint)


def test_rfc9380_p384_vector():
    """RFC 9380 J.3.1, P384_XMD:SHA-384_SSWU_RO_, msg = ""."""
    x, y = O.hash_to_curve(b"", b"QUUX-V01-CS02-with-P384_XMD:SHA-384_SSWU_RO_")
    assert x == 0xeb9fe1b4f4e14e7140803c1d99d0a93cd823d2b024040f9c067a8eca1f5a2eeac9ad604973527a356f3fa3aeff0e4d83
    assert y == 0x0c21708cff382b7f4643c07b105c2eaec2cead93a917d825601e63c8f21f6abd9abc22c93c2bed6f235954b25048bb1a


def test_context_string_follows_rfc9497():
    assert O.CONTEXT_STRING == b"OPRFV1-\x01-P384-SHA384"
    assert O.HASH_TO_GROUP_DST == b"HashToGroup-OPRFV1-\x01-P384-SHA384"


@pytest.mark.parametrize("k", [1, 2, 3, O.N - 1, O.N - 6, 0x1234567, "random"])
def test_scalar_multiplication_matches_cryptography(k):
    k = random.Random(1).randrange(1, O.N) if k == "random" else k
    assert O.public_key(k.to_bytes(48, "big")) == compressed_public_key(k)
    assert O.to_affine(O.jacobian_mul(k, O.G)) == O.mul(k, O.G) == O.mul_affine(k, O.G)


def test_recoding_is_exact():
    rng = random.Random(2)
    for k in [1, 3, O.N - 2, 2**383 + 1, 2**384 - 1] + [rng.randrange(1, O.N) | 1 for _ in range(20)]:
        digits = O.recode(k)
        assert len(digits) == O.DIGITS and digits[-1] > 0
        assert all(d % 2 == 1 and abs(d) < 16 for d in digits)
        assert sum(d << (4 * i) for i, d in enumerate(digits)) == k


def test_hash_to_group_times_k_is_ecdh():
    """The x of k HashToGroup(input) is the ECDH shared secret of k with the hashed point."""
    rng = random.Random(3)
    for _ in range(4):
        k = rng.randrange(1, O.N)
        element = O.serialize_element(O.hash_to_group(rng.randbytes(rng.randrange(40))))
        peer = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP384R1(), element)
        shared = ec.derive_private_key(k, ec.SECP384R1()).exchange(ec.ECDH(), peer)
        assert shared == O.mul(k, O.deserialize_element(element))[0].to_bytes(48, "big")


def test_sswu_straight_line_equals_the_definition():
    rng = random.Random(4)
    branches = set()
    for u in [0, 1, O.P - 1] + [rng.randrange(O.P) for _ in range(40)]:
        x, y, square = O.map_to_curve_sswu_generic(u)
        assert O.map_to_curve_sswu(u) == (x, y) and O.on_curve((x, y))
        branches.add(square)
    assert branches == {True, False}


def test_oprf_roundtrip():
    """oprfRoundtrip: Finalize(Blind -> BlindEvaluate -> unblind) equals Evaluate; two blinds differ, outputs agree."""
    key = random.Random(5).randrange(1, O.N).to_bytes(48, "big")
    for data in (b"", b"keyword", bytes(range(200))):
        r1, blinded1 = O.blind(data)
        r2, blinded2 = O.blind(data)
        assert blinded1 != blinded2
        out1 = O.finalize(data, r1, O.blind_evaluate(key, blinded1))
        out2 = O.finalize(data, r2, O.blind_evaluate(key, blinded2))
        assert out1 == out2 == O.evaluate(key, data)


@pytest.mark.parametrize("bad", [0, O.N, O.N + 1, 2**384 - 1])
def test_key_range(bad):
    with pytest.raises(ValueError):
        O.evaluate(bad.to_bytes(48, "big"), b"x")


def test_processed_rows_open():
    """The reference's database test: every sealed row opens with AESGCM(h[24:]) and nonce h[:12], and not with a
    13-byte nonce."""
    rng = random.Random(6)
    key = rng.randrange(1, O.N).to_bytes(48, "big")
    rows = [(rng.randbytes(rng.randrange(1, 20)), rng.randbytes(rng.randrange(0, 50))) for _ in range(10)]
    for (keyword, value), (new_keyword, sealed) in zip(rows, O.symmetric_pir_process(key, rows)):
        h = O.evaluate(key, keyword)
        assert new_keyword == h[:16] and len(sealed) == len(value) + 16
        assert AESGCM(h[24:]).decrypt(h[:12], sealed, None) == value
        with pytest.raises(InvalidTag):
            AESGCM(h[24:]).decrypt(h[:13], sealed, None)
