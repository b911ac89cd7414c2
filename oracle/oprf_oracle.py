"""Restatement of the reference's symmetric keyword PIR processing (SymmetricPir/SymmetricPirDatabase.swift:186-211) in
Python integers and hashlib, for the tests:

  - P-384 (SEC 2 / FIPS 186-5) in affine and Jacobian coordinates;
  - RFC 9380 expand_message_xmd (SHA-384), hash_to_field, simplified SWU with Z = -12 and hash_to_curve
    (suite P384_XMD:SHA-384_SSWU_RO_);
  - RFC 9497 VOPRF mode over P384-SHA384: Evaluate, and Blind / BlindEvaluate / Finalize without the DLEQ proof;
  - symmetricPIRProcess, with cryptography's AESGCM for the AES-GCM-192 seal (the only thing it is used for here).

CONTEXT_STRING follows RFC 9497's text ("OPRFV1-" || I2OSP(mode, 1) || "-" || identifier, mode 0x01 for VOPRF); it
has not been checked against swift-crypto's P384._VOPRF bytes, which no vector on hand pins.
"""
from __future__ import annotations

import hashlib
import secrets
from typing import List, Optional, Sequence, Tuple

P = 2**384 - 2**128 - 2**96 + 2**32 - 1
N = 0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973
A = P - 3
B = 0xb3312fa7e23ee7e4988e056be3f82d19181d9c6efe8141120314088f5013875ac656398d8a2ed19d2a85c8edd3ec2aef
GX = 0xaa87ca22be8b05378eb1c71ef320ad746e1d3b628ba79b9859f741e082542a385502f25dbf55296c3a545e3872760ab7
GY = 0x3617de4a96262c6f5d9e98bf9292dc29f8f41dbd289a147ce9da3113b5f0b8c00a60b1ce1d7e819d7a431d7c90ea0e5f
G = (GX, GY)
Z_SSWU = P - 12

CONTEXT_STRING = b"OPRFV1-" + bytes([0x01]) + b"-P384-SHA384"
HASH_TO_GROUP_DST = b"HashToGroup-" + CONTEXT_STRING
KEY_BYTES, ELEMENT_BYTES, OUTPUT_BYTES = 48, 49, 48
KEYWORD_BYTES, NONCE_BYTES, AES_KEY_BYTES, TAG_BYTES = 16, 12, 24, 16

Point = Optional[Tuple[int, int]]  # affine; None is the identity


# ---------------------------------------------------------------- field
def inv(a: int) -> int:
    return pow(a, P - 2, P)


def is_square(a: int) -> bool:
    return a % P == 0 or pow(a, (P - 1) // 2, P) == 1


def sqrt(a: int) -> int:
    return pow(a, (P + 1) // 4, P)  # p = 3 mod 4


def sgn0(a: int) -> int:
    return a % P & 1


def sqrt_ratio(u: int, v: int) -> Tuple[bool, int]:
    """RFC 9380 F.2.1.2 (q = 3 mod 4): (True, sqrt(u/v)) or (False, sqrt(Z u/v))."""
    c1 = (P - 3) // 4
    c2 = sqrt(-Z_SSWU % P)
    tv1 = v * v % P
    tv2 = u * v % P
    tv1 = tv1 * tv2 % P
    y1 = pow(tv1, c1, P) * tv2 % P
    y2 = y1 * c2 % P
    is_qr = y1 * y1 % P * v % P == u % P
    return is_qr, (y1 if is_qr else y2)


# ---------------------------------------------------------------- group, affine
def on_curve(pt: Point) -> bool:
    if pt is None:
        return True
    x, y = pt
    return (y * y - (x * x * x + A * x + B)) % P == 0


def add(p1: Point, p2: Point) -> Point:
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = (3 * x1 * x1 + A) * inv(2 * y1) % P
    else:
        lam = (y2 - y1) * inv(x2 - x1) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def neg(pt: Point) -> Point:
    return None if pt is None else (pt[0], -pt[1] % P)


def mul(k: int, pt: Point) -> Point:
    """k * pt by binary double-and-add over Jacobian points, one inversion at the end."""
    k %= N
    out = (1, 1, 0)
    base = to_jacobian(pt)
    for bit in bin(k)[2:]:
        out = jacobian_double(out)
        if bit == "1":
            out = jacobian_add(out, base)
    return to_affine(out)


def mul_affine(k: int, pt: Point) -> Point:
    """k * pt by double-and-add over affine points (slow; checks the Jacobian formulas)."""
    k %= N
    out: Point = None
    for bit in bin(k)[2:]:
        out = add(out, out)
        if bit == "1":
            out = add(out, pt)
    return out


# ---------------------------------------------------------------- group, Jacobian (a = -3)
def jacobian_double(pt):
    x1, y1, z1 = pt
    if z1 == 0 or y1 == 0:
        return (1, 1, 0)
    delta = z1 * z1 % P
    gamma = y1 * y1 % P
    beta = x1 * gamma % P
    alpha = 3 * (x1 - delta) * (x1 + delta) % P
    x3 = (alpha * alpha - 8 * beta) % P
    z3 = ((y1 + z1) ** 2 - gamma - delta) % P
    y3 = (alpha * (4 * beta - x3) - 8 * gamma * gamma) % P
    return x3, y3, z3


def jacobian_add(p1, p2):
    x1, y1, z1 = p1
    x2, y2, z2 = p2
    if z1 == 0:
        return p2
    if z2 == 0:
        return p1
    z1z1, z2z2 = z1 * z1 % P, z2 * z2 % P
    u1, u2 = x1 * z2z2 % P, x2 * z1z1 % P
    s1, s2 = y1 * z2 * z2z2 % P, y2 * z1 * z1z1 % P
    h = (u2 - u1) % P
    r = 2 * (s2 - s1) % P
    if h == 0:
        return jacobian_double(p1) if r == 0 else (1, 1, 0)
    i = 4 * h * h % P
    j = h * i % P
    v = u1 * i % P
    x3 = (r * r - j - 2 * v) % P
    y3 = (r * (v - x3) - 2 * s1 * j) % P
    z3 = ((z1 + z2) ** 2 - z1z1 - z2z2) * h % P
    return x3, y3, z3


def to_jacobian(pt: Point):
    return (1, 1, 0) if pt is None else (pt[0], pt[1], 1)


def to_affine(pt) -> Point:
    x, y, z = pt
    if z % P == 0:
        return None
    zi = inv(z)
    return x * zi * zi % P, y * zi * zi * zi % P


DIGITS = 96


def recode(k: int, window: int = 4) -> List[int]:
    """The regular signed-window recoding of an odd k < 2^384: 96 digits d_0 .. d_95, each odd with |d| < 2^window,
    and k = sum d_i 2^(window i).  The top digit is positive."""
    assert k & 1 and 0 < k < 1 << (DIGITS * window)
    digits = []
    for _ in range(DIGITS - 1):
        d = (k % (1 << (window + 1))) - (1 << window)
        digits.append(d)
        k = (k - d) >> window
    assert 0 < k < 1 << window
    digits.append(k)
    return digits


def jacobian_mul(k: int, pt: Point):
    """k * pt through the fixed-window ladder the device runs: k made odd (k or n - k, then the result negated), recoded
    into 4-bit signed odd digits, 4 doublings and one addition of a table entry per digit."""
    k %= N
    flip = k % 2 == 0
    if flip:
        k = N - k
    digits = recode(k)
    base = to_jacobian(pt)
    twice = jacobian_double(base)
    table = [base]
    for _ in range(7):
        table.append(jacobian_add(table[-1], twice))
    acc = table[(digits[-1] - 1) // 2]
    for d in reversed(digits[:-1]):
        for _ in range(4):
            acc = jacobian_double(acc)
        x, y, z = table[(abs(d) - 1) // 2]
        acc = jacobian_add(acc, (x, y if d > 0 else -y % P, z))
    if flip:
        acc = (acc[0], -acc[1] % P, acc[2])
    return acc


# ---------------------------------------------------------------- encoding
def i2osp(value: int, length: int) -> bytes:
    return value.to_bytes(length, "big")


def serialize_element(pt: Point) -> bytes:
    """SEC1 compressed form, 49 bytes (RFC 9497 SerializeElement for P-384)."""
    if pt is None:
        raise ValueError("the identity has no encoding")
    x, y = pt
    return bytes([2 | (y & 1)]) + i2osp(x, 48)


def deserialize_element(data: bytes) -> Point:
    if len(data) != ELEMENT_BYTES or data[0] not in (2, 3):
        raise ValueError("not a compressed P-384 point")
    x = int.from_bytes(data[1:], "big")
    if x >= P:
        raise ValueError("x out of range")
    y2 = (x * x * x + A * x + B) % P
    if not is_square(y2):
        raise ValueError("not on the curve")
    y = sqrt(y2)
    if y & 1 != data[0] & 1:
        y = P - y
    return x, y


# ---------------------------------------------------------------- RFC 9380 hash_to_curve
def expand_message_xmd(msg: bytes, dst: bytes, len_in_bytes: int) -> bytes:
    """RFC 9380 5.3.1 with SHA-384 (b_in_bytes 48, s_in_bytes 128)."""
    b_in_bytes, s_in_bytes = 48, 128
    ell = -(-len_in_bytes // b_in_bytes)
    assert ell <= 255 and len_in_bytes <= 65535 and len(dst) <= 255
    dst_prime = dst + i2osp(len(dst), 1)
    msg_prime = bytes(s_in_bytes) + msg + i2osp(len_in_bytes, 2) + i2osp(0, 1) + dst_prime
    b0 = hashlib.sha384(msg_prime).digest()
    blocks = [hashlib.sha384(b0 + i2osp(1, 1) + dst_prime).digest()]
    for i in range(2, ell + 1):
        mixed = bytes(a ^ b for a, b in zip(b0, blocks[-1]))
        blocks.append(hashlib.sha384(mixed + i2osp(i, 1) + dst_prime).digest())
    return b"".join(blocks)[:len_in_bytes]


def hash_to_field(msg: bytes, dst: bytes, count: int = 2) -> List[int]:
    """RFC 9380 5.2 with L = 72 (k = 192), m = 1."""
    length = 72
    uniform = expand_message_xmd(msg, dst, count * length)
    return [int.from_bytes(uniform[length * i:length * (i + 1)], "big") % P for i in range(count)]


def map_to_curve_sswu(u: int) -> Tuple[int, int]:
    """RFC 9380 6.6.2 (simplified SWU, Z = -12), in the straight-line form of F.2."""
    tv1 = Z_SSWU * u * u % P
    tv2 = (tv1 * tv1 + tv1) % P
    tv3 = B * (tv2 + 1) % P
    tv4 = A * (Z_SSWU if tv2 == 0 else -tv2 % P) % P
    tv6 = tv4 * tv4 % P
    gx_num = (tv3 * tv3 + A * tv6) * tv3 % P
    tv6 = tv6 * tv4 % P
    gx_num = (gx_num + B * tv6) % P
    x = tv1 * tv3 % P
    is_gx1_square, y1 = sqrt_ratio(gx_num, tv6)
    y = tv1 * u % P * y1 % P
    if is_gx1_square:
        x, y = tv3, y1
    if sgn0(u) != sgn0(y):
        y = -y % P
    return x * inv(tv4) % P, y


def map_to_curve_sswu_generic(u: int) -> Tuple[int, int, bool]:
    """The same map by its defining formulas (RFC 9380 6.6.2): (x, y, gx1 is square)."""
    z = Z_SSWU
    den = (z * z * pow(u, 4, P) + z * u * u) % P
    tv1 = 0 if den == 0 else inv(den)
    x1 = (-B * inv(A)) * (1 + tv1) % P
    if tv1 == 0:
        x1 = B * inv(z * A) % P
    gx1 = (x1 ** 3 + A * x1 + B) % P
    x2 = z * u * u * x1 % P
    gx2 = (x2 ** 3 + A * x2 + B) % P
    square = is_square(gx1)
    x, y = (x1, sqrt(gx1)) if square else (x2, sqrt(gx2))
    if sgn0(u) != sgn0(y):
        y = -y % P
    return x, y, square


def hash_to_curve(msg: bytes, dst: bytes) -> Point:
    u0, u1 = hash_to_field(msg, dst)
    return add(map_to_curve_sswu(u0), map_to_curve_sswu(u1))  # cofactor 1


# ---------------------------------------------------------------- RFC 9497 VOPRF, P384-SHA384
def hash_to_group(data: bytes) -> Point:
    return hash_to_curve(data, HASH_TO_GROUP_DST)


def check_key(secret_key: bytes) -> int:
    if len(secret_key) != KEY_BYTES:
        raise ValueError(f"invalid OPRF key size {len(secret_key)}")
    k = int.from_bytes(secret_key, "big")
    if not 0 < k < N:
        raise ValueError("OPRF key out of range")
    return k


def public_key(secret_key: bytes) -> bytes:
    return serialize_element(mul(check_key(secret_key), G))


def finalize_hash(data: bytes, issued: bytes) -> bytes:
    return hashlib.sha384(i2osp(len(data), 2) + data + i2osp(len(issued), 2) + issued + b"Finalize").digest()


def evaluate(secret_key: bytes, data: bytes) -> bytes:
    """RFC 9497 3.3.1 Evaluate: SHA-384(I2OSP(len(input), 2) || input || I2OSP(49, 2) || k HashToGroup(input) ||
    "Finalize")."""
    k = check_key(secret_key)
    element = hash_to_group(data)
    if element is None:
        raise ValueError("InvalidInputError")
    return finalize_hash(data, serialize_element(mul(k, element)))


def blind(data: bytes, r: Optional[int] = None) -> Tuple[int, bytes]:
    r = r if r is not None else secrets.randbelow(N - 1) + 1
    return r, serialize_element(mul(r, hash_to_group(data)))


def blind_evaluate(secret_key: bytes, blinded: bytes) -> bytes:
    return serialize_element(mul(check_key(secret_key), deserialize_element(blinded)))


def finalize(data: bytes, r: int, evaluated: bytes) -> bytes:
    unblinded = mul(pow(r, N - 2, N), deserialize_element(evaluated))
    return finalize_hash(data, serialize_element(unblinded))


# ---------------------------------------------------------------- symmetricPIRProcess
def split_output(h: bytes) -> Tuple[bytes, bytes, bytes]:
    """(keyword', nonce, AES key) of an OPRF output: h[0:16], h[0:12], h[24:48] (SymmetricPirDatabase.swift:202-206)."""
    return h[:KEYWORD_BYTES], h[:NONCE_BYTES], h[-AES_KEY_BYTES:]


def seal(h: bytes, value: bytes) -> bytes:
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    _, nonce, key = split_output(h)
    return AESGCM(key).encrypt(nonce, bytes(value), None)  # ciphertext || 16-byte tag


def symmetric_pir_process(secret_key: bytes, rows: Sequence[Tuple[bytes, bytes]]) -> List[Tuple[bytes, bytes]]:
    out = []
    for keyword, value in rows:
        h = evaluate(secret_key, bytes(keyword))
        out.append((split_output(h)[0], seal(h, value)))
    return out
