"""CPU restatement of the reference's processed PNNS database file, for the tests: the protobuf message
apple.swift_homomorphic_encryption.pnns.v1.SerializedProcessedDatabase as ProcessedDatabase.serialize() and
PnnsConversion.swift's proto() build it and SwiftProtobuf writes it, and a parser for it.

    SerializedProcessedDatabase  1 plaintext_matrices  2 entry_ids (packed)  3 entry_metadatas  4 server_config
    SerializedPlaintextMatrix    1 num_rows  2 num_columns  3 plaintexts { 1 poly }  4 packing
    ServerConfig                 1 client_config  2 database_packing
    ClientConfig                 1 encryption_parameters  2 scaling_factor  3 query_packing  4 vector_dimension
                                 5 galois_elements (packed)  6 distance_metric  7 extra_plaintext_moduli (packed)
    MatrixPacking                oneof 1 dense_row {}  2 diagonal { 2 baby_step_giant_step { 1 2 3 } }  3 dense_column {}
    v1.EncryptionParameters      1 polynomial_degree  2 plaintext_modulus  3 coefficient_moduli (packed)
                                 4 error_std_dev  5 security_level  6 he_scheme

SwiftProtobuf writes fields in field-number order, omits proto3 zero scalars and enums, writes a set message even
when it is empty, and packs repeated scalars.  Each `poly` is the oracle's pinned PolyRq codec (serialize_poly) of an
Eval plaintext's L rows.  Configs are dicts keyed by the proto field names; a packing is ("denseRow",),
("denseColumn",) or ("diagonal", (vector_dimension, baby_step, giant_step))."""
from __future__ import annotations

import numpy as np

from oracle import pir_oracle as opir
from oracle import pnns_oracle as opnns

PACKINGS = {"denseRow": 1, "diagonal": 2, "denseColumn": 3}


class ProtoError(ValueError):
    pass


# ---- writing ---------------------------------------------------------------------------------------------------------

def varint(v: int) -> bytes:
    v = int(v) & ((1 << 64) - 1)
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def key(number: int, wire: int) -> bytes:
    return varint(number << 3 | wire)


def scalar(number: int, v: int) -> bytes:
    return key(number, 0) + varint(v) if v else b""


def message(number: int, body: bytes) -> bytes:
    return key(number, 2) + varint(len(body)) + body


def packed(number: int, values) -> bytes:
    values = list(values)
    return message(number, b"".join(varint(v) for v in values)) if values else b""


def encode_packing(packing) -> bytes:
    kind = packing[0]
    member = b""
    if kind == "diagonal":
        d, b, g = packing[1]
        member = message(2, scalar(1, d) + scalar(2, b) + scalar(3, g))
    return message(PACKINGS[kind], member)


def encode_encryption_parameters(p: dict) -> bytes:
    return (scalar(1, p["polynomial_degree"]) + scalar(2, p["plaintext_modulus"]) + packed(3, p["coefficient_moduli"]) +
            scalar(4, p.get("error_std_dev", 0)) + scalar(5, p.get("security_level", 0)) + scalar(6, p.get("he_scheme", 1)))


def encode_client_config(c: dict) -> bytes:
    return (message(1, encode_encryption_parameters(c["encryption_parameters"])) + scalar(2, c["scaling_factor"]) +
            message(3, encode_packing(c.get("query_packing", ("denseRow",)))) + scalar(4, c["vector_dimension"]) +
            packed(5, c.get("galois_elements", [])) + scalar(6, c.get("distance_metric", 0)) +
            packed(7, c.get("extra_plaintext_moduli", [])))


def encode_server_config(s: dict) -> bytes:
    return message(1, encode_client_config(s["client_config"])) + message(2, encode_packing(s["database_packing"]))


def encode_processed_database(matrices, entry_ids, entry_metadatas, server_config: dict) -> bytes:
    """matrices: dicts with num_rows, num_columns, plaintexts (the poly bytes of each) and packing."""
    out = bytearray()
    for m in matrices:
        body = scalar(1, m["num_rows"]) + scalar(2, m["num_columns"])
        body += b"".join(message(3, message(1, poly)) for poly in m["plaintexts"])
        body += message(4, encode_packing(m["packing"]))
        out += message(1, body)
    out += packed(2, entry_ids)
    out += b"".join(message(3, bytes(meta)) for meta in entry_metadatas)
    out += message(4, encode_server_config(server_config))
    return bytes(out)


# ---- the plaintexts, from the oracle ---------------------------------------------------------------------------------

def diagonal_polys(ctx, rows: int, cols: int, values, bsgs) -> list:
    """The poly bytes of PlaintextMatrix(.diagonal) over the oracle context `ctx` of values already in [0, t): the
    diagonal plaintexts, each converted to Eval over the ciphertext moduli and serialized."""
    moduli = ctx.moduli[:ctx.L]
    ob = opnns.BabyStepGiantStep(*bsgs)
    return [opir.serialize_poly(ctx.n, moduli, ctx.plaintext_to_eval(p))
            for p in opnns.diagonal_plaintexts(ctx, rows, cols, ob, values)]


def polys_from_resident(n: int, moduli, words: np.ndarray, rows: int, cols: int, bsgs) -> list:
    """The poly bytes of a resident [result][giant][baby] x L x N matrix, in the reference's plaintext order
    (index resultCount * (j + babyStep * g) + r is slot (r, g, j))."""
    dimension, baby, giant = bsgs
    results = -(-rows // n)
    words = np.asarray(words, dtype=np.uint64).reshape(results * giant * baby, len(moduli), n)
    out = []
    for p in range(dimension * results):
        r, d = p % results, p // results
        out.append(opir.serialize_poly(n, moduli, words[(r * giant + d // baby) * baby + d % baby]))
    return out


# ---- reading ---------------------------------------------------------------------------------------------------------

def read_varint(data: bytes, at: int, end: int):
    v = 0
    for k in range(10):
        if at >= end:
            raise ProtoError("truncated varint")
        b = data[at]
        at += 1
        v |= (b & 0x7F) << (7 * k)
        if not b & 0x80:
            return v & ((1 << 64) - 1), at
    raise ProtoError("varint longer than 10 bytes")


def fields(data: bytes, at: int = 0, end: int = None):
    """(number, wire, value) of every field of the message data[at:end]; value is an int or the payload bytes."""
    end = len(data) if end is None else end
    while at < end:
        k, at = read_varint(data, at, end)
        number, wire = k >> 3, k & 7
        if number == 0:
            raise ProtoError("field number 0")
        if wire == 0:
            v, at = read_varint(data, at, end)
        elif wire in (1, 5):
            size = 8 if wire == 1 else 4
            if end - at < size:
                raise ProtoError("truncated fixed field")
            v, at = int.from_bytes(data[at:at + size], "little"), at + size
        elif wire == 2:
            size, at = read_varint(data, at, end)
            if size > end - at:
                raise ProtoError("length runs past the end")
            v, at = data[at:at + size], at + size
        else:
            raise ProtoError(f"wire type {wire}")
        yield number, wire, v


def _repeated(wire, v, out):
    if wire == 0:
        out.append(v)
    elif wire == 2:
        at = 0
        while at < len(v):
            x, at = read_varint(v, at, len(v))
            out.append(x)
    else:
        raise ProtoError("wrong wire type")


def _single(msg, number, wire, v, name):
    if wire != 2:
        raise ProtoError(f"{name}: wrong wire type")
    if number in msg:
        raise ProtoError(f"{name}: a singular message given twice")
    msg[number] = v


def parse_packing(data: bytes):
    packing, seen = None, {}
    for number, wire, v in fields(data):
        if number in (1, 2, 3):
            _single(seen, number, wire, v, "MatrixPacking")
            kind = {1: "denseRow", 2: "diagonal", 3: "denseColumn"}[number]
            packing = (kind,)
            if kind == "diagonal":
                inner = {}
                for n2, w2, v2 in fields(v):
                    if n2 == 2:
                        _single(inner, n2, w2, v2, "MatrixPackingDiagonal")
                if 2 not in inner:
                    raise ProtoError("unsetField(diagonal.babyStepGiantStep)")
                steps = [0, 0, 0]
                for n3, w3, v3 in fields(inner[2]):
                    if n3 in (1, 2, 3):
                        steps[n3 - 1] = v3
                packing = (kind, tuple(steps))
    if packing is None:
        raise ProtoError("unsetOneof(matrixPackingType)")
    return packing


def parse_client_config(data: bytes) -> dict:
    msgs, out = {}, {"scaling_factor": 0, "vector_dimension": 0, "galois_elements": [], "distance_metric": 0,
                     "extra_plaintext_moduli": []}
    for number, wire, v in fields(data):
        if number in (1, 3):
            _single(msgs, number, wire, v, "ClientConfig")
        elif number in (2, 4, 6):
            out[{2: "scaling_factor", 4: "vector_dimension", 6: "distance_metric"}[number]] = v
        elif number == 5:
            _repeated(wire, v, out["galois_elements"])
        elif number == 7:
            _repeated(wire, v, out["extra_plaintext_moduli"])
    if 1 not in msgs:
        raise ProtoError("unsetField(encryptionParameters)")
    p = {"polynomial_degree": 0, "plaintext_modulus": 0, "coefficient_moduli": [], "error_std_dev": 0,
         "security_level": 0, "he_scheme": 0}
    names = {1: "polynomial_degree", 2: "plaintext_modulus", 4: "error_std_dev", 5: "security_level", 6: "he_scheme"}
    for number, wire, v in fields(msgs[1]):
        if number == 3:
            _repeated(wire, v, p["coefficient_moduli"])
        elif number in names:
            p[names[number]] = v
    if p["he_scheme"] == 2:
        raise ProtoError("invalidScheme")
    out["encryption_parameters"] = p
    out["query_packing"] = parse_packing(msgs.get(3, b""))
    return out


def parse_server_config(data: bytes) -> dict:
    msgs = {}
    for number, wire, v in fields(data):
        if number in (1, 2):
            _single(msgs, number, wire, v, "ServerConfig")
    if 1 not in msgs:
        raise ProtoError("unsetField(clientConfig)")
    return {"client_config": parse_client_config(msgs[1]), "database_packing": parse_packing(msgs.get(2, b""))}


def parse_processed_database(data: bytes) -> dict:
    data = bytes(data)
    out = {"matrices": [], "entry_ids": [], "entry_metadatas": []}
    config = {}
    for number, wire, v in fields(data):
        if number == 1:
            m = {"num_rows": 0, "num_columns": 0, "plaintexts": []}
            packing = {}
            for n2, w2, v2 in fields(v):
                if n2 in (1, 2):
                    m["num_rows" if n2 == 1 else "num_columns"] = v2
                elif n2 == 3:
                    poly = b""
                    for n3, w3, v3 in fields(v2):
                        if n3 == 1:
                            poly = v3
                    m["plaintexts"].append(poly)
                elif n2 == 4:
                    _single(packing, n2, w2, v2, "SerializedPlaintextMatrix")
            m["packing"] = parse_packing(packing.get(4, b""))
            out["matrices"].append(m)
        elif number == 2:
            _repeated(wire, v, out["entry_ids"])
        elif number == 3:
            out["entry_metadatas"].append(bytes(v))
        elif number == 4:
            _single(config, number, wire, v, "SerializedProcessedDatabase")
    if 4 not in config:
        raise ProtoError("unsetField(serverConfig)")
    out["server_config"] = parse_server_config(config[4])
    return out
