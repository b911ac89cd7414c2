"""An independent restatement of the PNNS protobuf messages, written from the reference's .proto files
(pnns/v1/pnns.proto, pnns/v1/pnns_matrix_packing.proto, api/pnns/v1/pnns.proto, api/shared/v1/api_shared.proto) and from
PnnsConversion.swift and PnnsConversionApi.swift.  Encoders give SwiftProtobuf's bytes (fields in number order, proto3
zero scalars omitted, set messages written even when empty, repeated scalars packed, every element of a repeated bytes
field written); the ciphertexts are those of tests/pir_proto_ref.py.

    SerializedCiphertextMatrix  1 num_rows  2 num_columns  3 ciphertexts  4 packing
    MatrixPacking               oneof 1 dense_row {}  2 diagonal { 2 baby_step_giant_step }  3 dense_column {}
    PNNSRequest                 1 shard_indices (packed uint32)  2 query (matrices)  3 evaluation_key_metadata
                                { 1 timestamp  2 identifier }  4 config_id  5 evaluation_key { 1 metadata
                                2 evaluation_key }  6 shard_ids
    PNNSShardResponse           1 reply (matrices)  2 entry_ids (packed uint64)  3 entry_metadatas"""
import pir_proto_ref as pir
from pir_proto_ref import LEN, ProtoError, field_bytes, field_scalar, fields, packed

DENSE_ROW, DIAGONAL, DENSE_COLUMN = 1, 2, 3


def encode_packing(kind):
    return field_bytes(kind, b"")


def encode_matrix(rows, columns, cts, packing):
    """SerializedCiphertextMatrix.proto(): cts as pir_proto_ref ciphertexts; packing None leaves the field unset."""
    return (field_scalar(1, rows) + field_scalar(2, columns) +
            b"".join(field_bytes(3, pir.encode_ciphertext(ct)) for ct in cts) +
            (field_bytes(4, encode_packing(packing)) if packing is not None else b""))


def encode_pnns_request(query, shard_indices=(), metadata=None, config_id=b"", evaluation_key=None, key_metadata=None,
                        shard_ids=()):
    """query: encoded matrices, one per plaintext modulus; metadata / key_metadata: (timestamp, identifier) of
    evaluation_key_metadata / evaluation_key.metadata; evaluation_key: SerializedEvaluationKey bytes."""
    out = packed(1, list(shard_indices)) + b"".join(field_bytes(2, m) for m in query)
    if metadata is not None:
        out += field_bytes(3, field_scalar(1, metadata[0]) + (field_bytes(2, metadata[1]) if metadata[1] else b""))
    out += field_bytes(4, config_id) if config_id else b""
    if evaluation_key is not None:
        inner = b""
        if key_metadata is not None:
            inner += field_bytes(1, field_scalar(1, key_metadata[0]) +
                                 (field_bytes(2, key_metadata[1]) if key_metadata[1] else b""))
        inner += field_bytes(2, evaluation_key)
        out += field_bytes(5, inner)
    return out + b"".join(field_bytes(6, s.encode()) for s in shard_ids)


def encode_shard_response(matrices, rows, columns, entry_ids, entry_metadatas):
    """Response.proto(): matrices [(replies [(poly0, poly1)], skips)] per plaintext modulus, each .denseColumn of rows x
    columns with .full ciphertexts (forDecryption), then the ids and metadata."""
    out = b""
    for replies, skips in matrices:
        cts = [("full", pir.full_polys(p0, p1), list(skips), 1) for p0, p1 in replies]
        out += field_bytes(1, encode_matrix(rows, columns, cts, DENSE_COLUMN))
    return out + packed(2, list(entry_ids)) + b"".join(field_bytes(3, m) for m in entry_metadatas)


def parse_matrix(b, begin, end, poly_bytes=None):
    """(rows, columns, packing, [ciphertext]) with ciphertexts parsed over poly_bytes, or their (begin, end) without."""
    rows = columns = 0
    packing, cts, seen_packing = 0, [], False
    for number, wire, v in fields(b, begin, end):
        if number in (1, 2):
            pir.expect(wire, 0)
            rows, columns = (v, columns) if number == 1 else (rows, v)
        elif number == 3:
            pir.expect(wire, LEN)
            cts.append(pir.parse_ciphertext(b, *v, poly_bytes) if poly_bytes else v)
        elif number == 4:
            pir.expect(wire, LEN)
            if seen_packing:
                raise ProtoError("invalid", "MatrixPacking given twice")
            seen_packing, packing = True, 0
            seen = set()
            for n2, w2, v2 in fields(b, *v):
                if n2 in (1, 2, 3):
                    pir.expect(w2, LEN)
                    if n2 in seen:
                        raise ProtoError("invalid", "a oneof member given twice")
                    seen.add(n2)
                    packing = n2
    return rows & 0xFFFFFFFF, columns & 0xFFFFFFFF, packing, cts


def parse_pnns_request(b):
    """Every field of a PNNSRequest: shardIndices, query (each matrix's (begin, end)), configId, keyTimestamp /
    keyIdentifier (evaluation_key_metadata, else evaluation_key.metadata), evaluationKey ((begin, end) or None),
    shardIds."""
    out = dict(shardIndices=[], query=[], configId=b"", keyTimestamp=None, keyIdentifier=None, evaluationKey=None,
               shardIds=[])
    inner_metadata = None

    def metadata(begin, end):
        ts, ident = 0, b""
        for number, wire, v in fields(b, begin, end):
            if number == 1:
                pir.expect(wire, 0)
                ts = v
            elif number == 2:
                pir.expect(wire, LEN)
                ident = b[v[0]:v[1]]
        return ts, ident

    for number, wire, v in fields(b):
        if number == 1:
            if wire == 0:
                out["shardIndices"].append(v)
            else:
                pir.expect(wire, LEN)
                at = v[0]
                while at < v[1]:
                    x, at = pir.read_varint(b, at, v[1])
                    out["shardIndices"].append(x)
        elif number == 2:
            pir.expect(wire, LEN)
            out["query"].append(v)
        elif number == 3:
            pir.expect(wire, LEN)
            out["keyTimestamp"], out["keyIdentifier"] = metadata(*v)
        elif number == 4:
            pir.expect(wire, LEN)
            out["configId"] = b[v[0]:v[1]]
        elif number == 5:
            pir.expect(wire, LEN)
            out["evaluationKey"] = (v[0], v[0])
            for n2, w2, v2 in fields(b, *v):
                if n2 == 1:
                    pir.expect(w2, LEN)
                    inner_metadata = metadata(*v2)
                elif n2 == 2:
                    pir.expect(w2, LEN)
                    out["evaluationKey"] = v2
        elif number == 6:
            pir.expect(wire, LEN)
            out["shardIds"].append(b[v[0]:v[1]].decode())
    if out["keyTimestamp"] is None and inner_metadata is not None:
        out["keyTimestamp"], out["keyIdentifier"] = inner_metadata
    return out


def parse_shard_response(b, poly_bytes):
    """([(rows, columns, packing, [ciphertext])], entry ids, entry metadatas)."""
    matrices, ids, metadatas = [], [], []
    for number, wire, v in fields(b):
        if number == 1:
            pir.expect(wire, LEN)
            matrices.append(parse_matrix(b, *v, poly_bytes))
        elif number == 2:
            if wire == 0:
                ids.append(v)
            else:
                pir.expect(wire, LEN)
                at = v[0]
                while at < v[1]:
                    x, at = pir.read_varint(b, at, v[1])
                    ids.append(x)
        elif number == 3:
            pir.expect(wire, LEN)
            metadatas.append(b[v[0]:v[1]])
    return matrices, ids, metadatas
