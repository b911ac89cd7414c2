"""An independent restatement of the PIR protobuf messages, written from the reference's .proto files
(v1/he.proto, pir/v1/pir.proto, api/pir/v1/pir.proto, api/shared/v1/api_shared.proto) and from ConversionHe.swift,
PirConversion.swift, PirConversionApi.swift and Serialize.swift.  Encoders give SwiftProtobuf's bytes (fields in number
order, proto3 zero scalars omitted, set messages written even when empty, repeated scalars packed); parsers refuse what
the library refuses, raising ProtoError(kind, what) with kind "invalid" or "unsupported".

    SerializedCiphertext     oneof 1 seeded { 1 poly0  2 seed }  2 full { 1 polys  2 skip_lsbs  3 correction_factor }
    SerializedCiphertextVec  1 ciphertexts
    SerializedKeySwitchKey   1 key_switch_key (SerializedCiphertextVec)
    SerializedEvaluationKey  1 galois_key { 1 map<uint64, SerializedKeySwitchKey> }  2 relin_key { 1 relin_key }
    EncryptedIndices         1 ciphertexts  2 num_pir_calls
    PIRRequest               1 shard_index  2 query  3 evaluation_key_metadata { 1 timestamp  2 identifier }
                             4 configuration_hash  5 shard_id  6 evaluation_key { 1 metadata  2 evaluation_key }
    PIRResponse              1 replies (SerializedCiphertextVec)  2 stash

Ciphertexts are ("seeded", poly0, seed) or ("full", polys, skip_lsbs, correction_factor), polys being
Serialize.serializePolys' bytes: UInt16 little-endian count, then the packed polynomials."""
import struct


class ProtoError(ValueError):
    def __init__(self, kind, what):
        super().__init__(f"{kind}: {what}")
        self.kind, self.what = kind, what


VARINT, FIXED64, LEN, FIXED32 = 0, 1, 2, 5


# ---- encoding ---------------------------------------------------------------------------------------------------------

def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def key(number, wire):
    return varint(number << 3 | wire)


def field_bytes(number, body):
    return key(number, LEN) + varint(len(body)) + bytes(body)


def field_scalar(number, v):
    return key(number, VARINT) + varint(v) if v else b""


def packed(number, values):
    return field_bytes(number, b"".join(varint(v) for v in values)) if values else b""


def full_polys(*polys):
    return struct.pack("<H", len(polys)) + b"".join(polys)


def encode_ciphertext(ct):
    if ct[0] == "seeded":
        _, poly0, seed = ct
        inner = (field_bytes(1, poly0) if poly0 else b"") + (field_bytes(2, seed) if seed else b"")
        return field_bytes(1, inner)
    _, polys, skips, correction = ct
    inner = (field_bytes(1, polys) if polys else b"") + packed(2, skips) + field_scalar(3, correction)
    return field_bytes(2, inner)


def encode_ciphertext_vec(cts):
    return b"".join(field_bytes(1, encode_ciphertext(ct)) for ct in cts)


def encode_encrypted_indices(cts, num_pir_calls):
    return b"".join(field_bytes(1, encode_ciphertext(ct)) for ct in cts) + field_scalar(2, num_pir_calls)


def encode_key_switch_key(cts):
    return field_bytes(1, encode_ciphertext_vec(cts))


def encode_evaluation_key(galois, relin=None):
    """galois: [(element, [ciphertexts])] in map order (None: galois_key unset); relin: [ciphertexts] or None."""
    out = b""
    if galois is not None:
        entries = b"".join(field_bytes(1, field_scalar(1, e) + field_bytes(2, encode_key_switch_key(cts)))
                           for e, cts in galois)
        out += field_bytes(1, entries)
    if relin is not None:
        out += field_bytes(2, field_bytes(1, encode_key_switch_key(relin)))
    return out


def encode_pir_request(shard_index=0, query=None, metadata=None, configuration_hash=b"", shard_id=None,
                       evaluation_key=None, key_metadata=None):
    """query / evaluation_key: message bytes; metadata / key_metadata: (timestamp, identifier)."""
    def md(m):
        return field_scalar(1, m[0]) + (field_bytes(2, m[1]) if m[1] else b"")

    out = field_scalar(1, shard_index)
    if query is not None:
        out += field_bytes(2, query)
    if metadata is not None:
        out += field_bytes(3, md(metadata))
    if configuration_hash:
        out += field_bytes(4, configuration_hash)
    if shard_id is not None:
        out += field_bytes(5, shard_id.encode())
    if evaluation_key is not None or key_metadata is not None:
        body = (field_bytes(1, md(key_metadata)) if key_metadata is not None else b"")
        body += field_bytes(2, evaluation_key) if evaluation_key is not None else b""
        out += field_bytes(6, body)
    return out


def encode_pir_response(replies, skips):
    """replies: [[(poly0 bytes, poly1 bytes)] per chunk] per index -> Response.proto() with .full ciphertexts."""
    return b"".join(field_bytes(1, encode_ciphertext_vec([("full", full_polys(p0, p1), list(skips), 1)
                                                          for p0, p1 in reply]))
                    for reply in replies)


# ---- parsing ----------------------------------------------------------------------------------------------------------

def read_varint(b, at, end):
    v = 0
    for k in range(10):
        if at >= end:
            raise ProtoError("invalid", "truncated varint")
        byte = b[at]
        at += 1
        v |= (byte & 0x7F) << (7 * k)
        if not byte & 0x80:
            return v, at
    raise ProtoError("invalid", "varint longer than 10 bytes")


def fields(b, begin=0, end=None):
    """(number, wire, value) with value an int (varint / fixed) or (begin, end) for LEN."""
    end = len(b) if end is None else end
    at = begin
    while at < end:
        k, at = read_varint(b, at, end)
        number, wire = k >> 3, k & 7
        if number == 0 or k >> 32:
            raise ProtoError("invalid", f"field number {number}")
        if wire == VARINT:
            v, at = read_varint(b, at, end)
            yield number, wire, v
        elif wire in (FIXED64, FIXED32):
            size = 8 if wire == FIXED64 else 4
            if end - at < size:
                raise ProtoError("invalid", "truncated fixed field")
            yield number, wire, int.from_bytes(b[at:at + size], "little")
            at += size
        elif wire == LEN:
            size, at = read_varint(b, at, end)
            if size > end - at:
                raise ProtoError("invalid", "length past the message")
            yield number, wire, (at, at + size)
            at += size
        elif wire in (3, 4):
            raise ProtoError("invalid", "group")
        else:
            raise ProtoError("invalid", f"wire type {wire}")


def expect(wire, want):
    if wire != want:
        raise ProtoError("invalid", f"wire type {wire}, expected {want}")


def parse_ciphertext(b, begin, end, poly_bytes, key=False):
    """poly_bytes(skip) -> serialized size of one polynomial, or -1."""
    kind, span, seen = None, None, set()
    for number, wire, value in fields(b, begin, end):
        if number in (1, 2):
            expect(wire, LEN)
            if number in seen:
                raise ProtoError("invalid", "a singular message given twice")
            seen.add(number)
            kind, span = number, value
    if kind is None:
        raise ProtoError("invalid", "unsetOneof")
    if kind == 1:
        poly0, seed = b"", b""
        for number, wire, value in fields(b, *span):
            if number in (1, 2):
                expect(wire, LEN)
                if number == 1:
                    poly0 = b[value[0]:value[1]]
                else:
                    seed = b[value[0]:value[1]]
        if len(poly0) != poly_bytes(0):
            raise ProtoError("invalid", "serializedBufferSizeMismatch")
        if len(seed) != 32:
            raise ProtoError("invalid", "seed size")
        return ("seeded", bytes(poly0), bytes(seed))
    if key:
        raise ProtoError("unsupported", ".full key ciphertext")
    polys, skips, correction = b"", [], 0
    for number, wire, value in fields(b, *span):
        if number == 1:
            expect(wire, LEN)
            polys = b[value[0]:value[1]]
        elif number == 2:
            if wire == VARINT:
                skips.append(value)
            else:
                expect(wire, LEN)
                at = value[0]
                while at < value[1]:
                    v, at = read_varint(b, at, value[1])
                    skips.append(v)
            if len(skips) > 2:
                raise ProtoError("unsupported", "more than 2 skip_lsbs")
        elif number == 3:
            expect(wire, VARINT)
            correction = value
    if correction != 1:
        raise ProtoError("unsupported", "correction factor")
    if len(polys) < 2 or struct.unpack("<H", bytes(polys[:2]))[0] != 2:
        raise ProtoError("invalid", "polys")
    if skips and len(skips) != 2:
        raise ProtoError("invalid", "skip_lsbs count")
    skips = skips or [0, 0]
    sizes = [poly_bytes(s) for s in skips]
    if min(sizes) < 0:
        raise ProtoError("invalid", "invalidCoefficientPacking")
    if len(polys) != 2 + sum(sizes):
        raise ProtoError("invalid", "serializedBufferSizeMismatch")
    return ("full", bytes(polys), skips, correction)


def parse_encrypted_indices(b, poly_bytes):
    cts, calls = [], 0
    for number, wire, value in fields(b):
        if number == 1:
            expect(wire, LEN)
            cts.append(parse_ciphertext(b, *value, poly_bytes))
        elif number == 2:
            expect(wire, VARINT)
            calls = value
    return cts, calls


def parse_key_switch_key(b, begin, end, poly_bytes, count):
    cts, seen = [], False
    for number, wire, value in fields(b, begin, end):
        if number != 1:
            continue
        expect(wire, LEN)
        if seen:
            raise ProtoError("invalid", "a singular message given twice")
        seen = True
        for n2, w2, v2 in fields(b, *value):
            if n2 == 1:
                expect(w2, LEN)
                cts.append(parse_ciphertext(b, *v2, poly_bytes, key=True))
    if len(cts) != count:
        raise ProtoError("invalid", "key switching key ciphertext count")
    return cts


def parse_evaluation_key(b, poly_bytes, count):
    """-> ({element: [ciphertexts]} in map order, [ciphertexts] or None)."""
    galois, relin, seen = {}, None, set()
    for number, wire, value in fields(b):
        if number not in (1, 2):
            continue
        expect(wire, LEN)
        if number in seen:
            raise ProtoError("invalid", "a singular message given twice")
        seen.add(number)
        if number == 1:
            for n2, w2, entry in fields(b, *value):
                if n2 != 1:
                    continue
                expect(w2, LEN)
                element, span, has = 0, (entry[0], entry[0]), False
                for n3, w3, v3 in fields(b, *entry):
                    if n3 == 1:
                        expect(w3, VARINT)
                        element = v3
                    elif n3 == 2:
                        expect(w3, LEN)
                        if has:
                            raise ProtoError("invalid", "a singular message given twice")
                        has, span = True, v3
                if element in galois:
                    raise ProtoError("invalid", "repeated Galois element")
                galois[element] = parse_key_switch_key(b, *span, poly_bytes, count)
        else:
            span, has = (value[0], value[0]), False
            for n2, w2, v2 in fields(b, *value):
                if n2 == 1:
                    expect(w2, LEN)
                    if has:
                        raise ProtoError("invalid", "a singular message given twice")
                    has, span = True, v2
            relin = parse_key_switch_key(b, *span, poly_bytes, count)
    return galois, relin


def parse_pir_request(b):
    out = {"shardIndex": 0, "shardId": None, "configurationHash": b"", "keyTimestamp": None, "keyIdentifier": None,
           "query": None, "evaluationKey": None}
    seen, inner_md = set(), None

    def metadata(span):
        ts, ident = 0, b""
        for number, wire, value in fields(b, *span):
            if number == 1:
                expect(wire, VARINT)
                ts = value
            elif number == 2:
                expect(wire, LEN)
                ident = bytes(b[value[0]:value[1]])
        out["keyTimestamp"], out["keyIdentifier"] = ts, ident

    for number, wire, value in fields(b):
        if number == 1:
            expect(wire, VARINT)
            out["shardIndex"] = value & 0xFFFFFFFF
        elif number in (2, 3, 6):
            expect(wire, LEN)
            if number in seen:
                raise ProtoError("invalid", "a singular message given twice")
            seen.add(number)
            if number == 2:
                out["query"] = (value[0], value[1] - value[0])
            elif number == 3:
                metadata(value)
            else:
                ek_seen = set()
                for n2, w2, v2 in fields(b, *value):
                    if n2 in (1, 2):
                        expect(w2, LEN)
                        if n2 in ek_seen:
                            raise ProtoError("invalid", "a singular message given twice")
                        ek_seen.add(n2)
                        if n2 == 1:
                            inner_md = v2
                        else:
                            out["evaluationKey"] = (v2[0], v2[1] - v2[0])
                if out["evaluationKey"] is None:
                    out["evaluationKey"] = (0, 0)
        elif number == 4:
            expect(wire, LEN)
            out["configurationHash"] = bytes(b[value[0]:value[1]])
        elif number == 5:
            expect(wire, LEN)
            out["shardId"] = bytes(b[value[0]:value[1]]).decode()
    if out["keyTimestamp"] is None and inner_md is not None:
        metadata(inner_md)
    return out


def parse_pir_response(b, poly_bytes):
    """-> [[("full", polys, skips, 1)] per chunk] per reply."""
    replies = []
    for number, wire, value in fields(b):
        if number != 1:
            continue
        expect(wire, LEN)
        reply = []
        for n2, w2, v2 in fields(b, *value):
            if n2 == 1:
                expect(w2, LEN)
                reply.append(parse_ciphertext(b, *v2, poly_bytes))
        replies.append(reply)
    return replies


def poly_sizes(n, bits):
    """poly_bytes(skip) for rows of `bits` bits at degree n (PolyContext.serializationByteCount)."""
    def size(skip):
        if any(skip >= w or skip < 0 for w in bits):
            return -1
        return sum((n * (w - skip) + 7) // 8 for w in bits)
    return size
