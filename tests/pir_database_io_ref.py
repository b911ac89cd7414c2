"""CPU restatement of the reference's processed-database file format, for the tests: ProcessedDatabase.serialize() and
init(from:context:) (IndexPirProtocol.swift:303-378) on top of the oracle's pinned PolyRq codec (serialize_poly,
load_poly).

    version byte (1) | plaintextCount (UInt32, little-endian) | per plaintext: tag 0 (nil), or tag 1 + PolyRq.serialize()

The load follows the reference: it checks the version and each tag, does not check residues against their moduli and
ignores trailing bytes.  Where the reference traps (a buffer that ends early) this raises corruptedData."""
from __future__ import annotations

from oracle import pir_oracle as opir

VERSION = 1


class DatabaseSerializationError(ValueError):
    pass


def serialize_processed_database(n: int, moduli, plaintexts) -> bytes:
    """plaintexts: a list of None (nil) or (L, N) Eval residues over the ciphertext moduli."""
    if all(p is None for p in plaintexts):
        raise DatabaseSerializationError("emptyDatabase")
    out = bytearray([VERSION]) + len(plaintexts).to_bytes(4, "little")
    for plaintext in plaintexts:
        if plaintext is None:
            out.append(0)
        else:
            out.append(1)
            out += opir.serialize_poly(n, moduli, plaintext)
    return bytes(out)


def from_processed(db) -> list:
    """An oracle ProcessedDatabase (plaintexts, present) as the list serialize_processed_database takes."""
    return [db.plaintexts[i] if db.present[i] else None for i in range(len(db.present))]


def load_processed_database(n: int, moduli, buffer: bytes) -> list:
    buffer = bytes(buffer)
    if not buffer:
        raise DatabaseSerializationError("corruptedData: empty buffer")
    if buffer[0] != VERSION:
        raise DatabaseSerializationError(
            f"invalidDatabaseSerializationVersion(serializationVersion: {buffer[0]}, expected: {VERSION})")
    if len(buffer) < 5:
        raise DatabaseSerializationError("corruptedData: header")
    count, offset = int.from_bytes(buffer[1:5], "little"), 5
    size = opir.serialization_byte_count(n, moduli)
    plaintexts = []
    for index in range(count):
        if offset >= len(buffer):
            raise DatabaseSerializationError(f"corruptedData: tag of plaintext {index}")
        tag = buffer[offset]
        offset += 1
        if tag == 0:
            plaintexts.append(None)
        elif tag == 1:
            if offset + size > len(buffer):
                raise DatabaseSerializationError(f"corruptedData: plaintext {index}")
            plaintexts.append(opir.load_poly(n, moduli, buffer[offset:offset + size]))
            offset += size
        else:
            raise DatabaseSerializationError(f"invalidDatabaseSerializationPlaintextTag(tag: {tag})")
    return plaintexts
