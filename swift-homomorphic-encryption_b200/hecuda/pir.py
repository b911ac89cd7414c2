"""hecuda.pir -- host-side mirror of the reference's MulPir index-PIR server over libhecuda (SURVEY.md 8f rank 3).

Names and argument meaning follow Sources/PrivateInformationRetrieval/IndexPir:

    IndexPirConfig, IndexPirParameter            IndexPirProtocol.swift:44-230
    MulPir.generateParameter / evaluationKeyConfig  MulPir.swift:37-109
    CoefficientPacking.bytesToCoefficients / coefficientsToBytes   HomomorphicEncryption/CoefficientPacking.swift
    MulPirServer.process / computeResponse       MulPir.swift:412-556, PirUtil.swift:490-568
    PirUtil.expand                               PirUtil.swift:321-355

    MulPirClient                                 MulPir.swift:119-290, PirUtil.swift:361-404
    ProcessedDatabaseWithParameters.validate     IndexPirProtocol.swift:420-484

The database stays resident in HBM (`ProcessedDatabase`); `computeResponse` is one C-ABI call per query.  The client
(key generation, query encryption, decryption, noise budgets) runs on the device too, so a processed database can be
validated the way the reference's PIRProcessDatabase does.  No CPU fallback: everything that touches ciphertexts or
plaintext polynomials runs in libhecuda.
"""
from __future__ import annotations

import ctypes as C
import os
import time
from dataclasses import dataclass, field
from enum import Enum
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np

from . import Bfv, Context, EvaluationKey, HeError, SecretKey, _check, _host, _ptr, load_library


class PirKeyCompressionStrategy(str, Enum):
    """PirKeyCompressionStrategy (IndexPirProtocol.swift:32-41)."""

    hybridCompression = "hybridCompression"
    maxCompression = "maxCompression"
    noCompression = "noCompression"


class PirError(ValueError):
    pass


def _ceil_log2(value: int) -> int:
    return max(0, (int(value) - 1).bit_length())


def _entry_size_encoding_width(entry_size: int) -> int:
    for width, limit in ((1, 1 << 8), (2, 1 << 16), (4, 1 << 32)):
        if entry_size < limit:
            return width
    return 8


class CoefficientPacking:
    """enum CoefficientPacking (CoefficientPacking.swift): big-endian bit-stream <-> fixed-width coefficients."""

    @staticmethod
    def bytesToCoefficients(data: bytes, bitsPerCoeff: int, decode: bool, skipLSBs: int = 0) -> np.ndarray:
        width = bitsPerCoeff - skipLSBs
        if not (bitsPerCoeff > 0 and width > 0 and skipLSBs >= 0):
            raise HeError(-1, f"invalidCoefficientPacking(bitsPerCoeff: {bitsPerCoeff}, skipLSBs: {skipLSBs})")
        total_bits = 8 * len(data)
        count = total_bits // width if decode else -(-total_bits // width)
        stream = int.from_bytes(bytes(data), "big")
        padded = count * width
        stream = stream << (padded - total_bits) if padded >= total_bits else stream >> (total_bits - padded)
        mask = (1 << width) - 1
        out = np.empty(count, dtype=np.uint64)
        for i in range(count - 1, -1, -1):
            out[i] = (stream & mask) << skipLSBs
            stream >>= width
        return out

    @staticmethod
    def coefficientsToBytes(coeffs: Sequence[int], bitsPerCoeff: int, skipLSBs: int = 0) -> bytes:
        width = bitsPerCoeff - skipLSBs
        if not (bitsPerCoeff > 0 and width > 0 and skipLSBs >= 0):
            raise HeError(-1, f"invalidCoefficientPacking(bitsPerCoeff: {bitsPerCoeff}, skipLSBs: {skipLSBs})")
        stream = 0
        for value in coeffs:
            stream = (stream << width) | ((int(value) >> skipLSBs) & ((1 << width) - 1))
        bits = len(coeffs) * width
        byte_count = -(-bits // 8)
        return (stream << (8 * byte_count - bits)).to_bytes(byte_count, "big")


def _pack_rows(pieces: List[Optional[bytes]], bits: int, degree: int):
    """Many byte strings -> (len(pieces), N) coefficient rows + presence flags (vectorised bytesToCoefficients)."""
    rows = np.zeros((len(pieces), degree), dtype=np.uint64)
    present = np.zeros(len(pieces), dtype=np.uint8)
    weights = (np.uint64(1) << np.arange(bits - 1, -1, -1, dtype=np.uint64))
    for i, piece in enumerate(pieces):
        if not piece:
            continue
        stream = np.unpackbits(np.frombuffer(piece, dtype=np.uint8))
        count = -(-stream.size // bits)
        if count > degree:
            raise PirError("plaintext bytes exceed bytesPerPlaintext")
        if count * bits != stream.size:
            stream = np.concatenate([stream, np.zeros(count * bits - stream.size, dtype=np.uint8)])
        values = stream.reshape(count, bits).astype(np.uint64) @ weights
        if values.any():
            rows[i, :count] = values
            present[i] = 1
    return rows, present


@dataclass
class IndexPirConfig:
    """IndexPirConfig (IndexPirProtocol.swift:44-104)."""

    entryCount: int
    entrySizeInBytes: int
    dimensionCount: int
    batchSize: int
    unevenDimensions: bool
    keyCompression: PirKeyCompressionStrategy
    encodingEntrySize: bool = False

    def __post_init__(self):
        if self.dimensionCount not in (1, 2):
            raise PirError(f"invalidDimensionCount(dimensionCount: {self.dimensionCount}, expected: [1, 2])")
        self.keyCompression = PirKeyCompressionStrategy(self.keyCompression)

    @property
    def entrySizeEncodingWidth(self) -> int:
        return _entry_size_encoding_width(self.entrySizeInBytes) if self.encodingEntrySize else 0

    @property
    def encodedEntrySize(self) -> int:
        return self.entrySizeEncodingWidth + self.entrySizeInBytes


@dataclass
class EvaluationKeyConfig:
    """EvaluationKeyConfig (Keys.swift:222): which Galois keys and whether a relinearization key are needed."""

    galoisElements: List[int] = field(default_factory=list)
    hasRelinearizationKey: bool = False


@dataclass
class IndexPirParameter:
    """IndexPirParameter (IndexPirProtocol.swift:160-230)."""

    entryCount: int
    entrySizeInBytes: int
    dimensions: List[int]
    batchSize: int
    evaluationKeyConfig: EvaluationKeyConfig
    encodingEntrySize: bool = False

    @property
    def entrySizeEncodingWidth(self) -> int:
        return _entry_size_encoding_width(self.entrySizeInBytes) if self.encodingEntrySize else 0

    @property
    def encodedEntrySize(self) -> int:
        return self.entrySizeEncodingWidth + self.entrySizeInBytes

    @property
    def dimensionCount(self) -> int:
        return len(self.dimensions)

    @property
    def expandedQueryCount(self) -> int:
        return int(sum(self.dimensions))


def bytesPerPlaintext(context) -> int:
    """Context.bytesPerPlaintext (EncryptionParameters.swift:103-110)."""
    return context.degree * (context.plaintextModulus.bit_length() - 1) // 8


class MulPir:
    """enum MulPir<Bfv<UInt64>>: IndexPirProtocol (MulPir.swift:24-115)."""

    @staticmethod
    def evaluationKeyConfig(expandedQueryCount: int, degree: int,
                            keyCompression: PirKeyCompressionStrategy) -> EvaluationKeyConfig:
        log_degree = degree.bit_length() - 1
        depth = _ceil_log2(min(expandedQueryCount, degree))
        smallest = log_degree - depth + 1
        compression = PirKeyCompressionStrategy(keyCompression)
        largest = log_degree if compression is PirKeyCompressionStrategy.noCompression else max(smallest, (log_degree + 2) // 2)
        powers = list(range(smallest, largest + 1))
        if compression is PirKeyCompressionStrategy.hybridCompression:
            extra = max(largest, (log_degree + largest + 1) // 2)
            if extra not in powers:
                powers.append(extra)
        return EvaluationKeyConfig([(1 << k) + 1 for k in powers], True)

    @staticmethod
    def generateParameter(config: IndexPirConfig, context) -> IndexPirParameter:
        per_plaintext_bytes = bytesPerPlaintext(context)
        encoded = config.encodedEntrySize
        if encoded <= per_plaintext_bytes:
            plaintexts = -(-config.entryCount // (per_plaintext_bytes // encoded))
        else:
            plaintexts = config.entryCount
        side = plaintexts
        if config.dimensionCount == 2:
            side = int(np.floor(np.sqrt(float(plaintexts))))
            while side * side > plaintexts:      # guard the floating-point root the way floor(root(x, 2)) behaves
                side -= 1
            while (side + 1) * (side + 1) <= plaintexts:
                side += 1
        dims = [side] * config.dimensionCount
        for i in range(len(dims)):
            if int(np.prod(dims, dtype=np.int64)) >= plaintexts:
                break
            dims[i] += 1
        if config.unevenDimensions and config.dimensionCount == 2:   # BFV only (MulPir.swift:56-71)
            def pow2(v):
                return 1 << _ceil_log2(v)
            limit = pow2(sum(dims) * config.batchSize)
            trial = list(dims)
            while pow2(sum(trial) * config.batchSize) <= limit:
                dims = list(trial)
                if trial[1] == 1:
                    break
                trial[1] -= 1
                trial[0] = -(-plaintexts // trial[1])
        evk = MulPir.evaluationKeyConfig(sum(dims) * config.batchSize, context.degree, config.keyCompression)
        return IndexPirParameter(config.entryCount, config.entrySizeInBytes, dims, config.batchSize, evk,
                                 config.encodingEntrySize)


def skipLSBsForDecryption(context) -> List[int]:
    """Bfv.skipLSBsForDecryption(for:) of a single-modulus ciphertext (Bfv+Decrypt.swift:51-110): how many low bits of
    poly 0 / poly 1 a reply may drop.  `context` needs degree, plaintextModulus, coefficientModuli."""
    q0, t = int(context.coefficientModuli[0]), int(context.plaintextModulus)
    l_prime = (q0 // t).bit_length() - 1 - 3 if q0 >= 2 * t else 0
    spread = int(8.0 * (2.0 * context.degree / 9.0) ** 0.5)
    poly0, poly1 = max(l_prime, 0), l_prime - (_ceil_log2(spread) if spread else 0)
    if poly1 <= 1:
        poly0, poly1 = max(l_prime + 1, 0), 0
    return [poly0, poly1]


class ProcessedDatabase:
    """ProcessedDatabase<Bfv<UInt64>> resident in HBM (IndexPirDatabase.swift): `count` optional Eval plaintexts."""

    def __init__(self, context: Context, plaintexts, present=None, evalFormat: bool = False):
        self.context = context
        rows = _host(plaintexts)
        words = context.degree * (context.L if evalFormat else 1)
        if rows.size % words:
            raise PirError("plaintext buffer has the wrong shape")
        self.count = rows.size // words
        flags = None
        if present is not None:
            flags = np.ascontiguousarray(np.asarray(present, dtype=np.uint8))
            if flags.size != self.count:
                raise PirError("presence flags have the wrong length")
        h = C.c_void_p()
        _check(load_library().hecuda_pir_database_create(context._h, _ptr(rows), 1 if evalFormat else 0,
                                                        flags.ctypes.data_as(C.c_void_p) if flags is not None else None,
                                                        self.count, C.byref(h)))
        self._h = h

    @classmethod
    def _adopt(cls, context: Context, handle: C.c_void_p, count: int) -> "ProcessedDatabase":
        db = cls.__new__(cls)
        db.context, db.count, db._h = context, count, handle
        return db

    def deviceBuffer(self):
        """(device pointer, bytes) of the resident rows: uint32 words when every ciphertext modulus is below 2^31."""
        p, n = C.c_void_p(), C.c_uint64(0)
        _check(load_library().hecuda_pir_database_device_buffer(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def presentFlags(self) -> np.ndarray:
        """The resident presence flags (count,): 0 for a nil plaintext the scan skips."""
        out = np.empty(self.count, dtype=np.uint8)
        _check(load_library().hecuda_pir_database_present(self._h, _ptr(out), self.count))
        return out

    def serializationByteCount(self) -> int:
        """ProcessedDatabase.serializationByteCount() (IndexPirProtocol.swift:336-348); HeError("emptyDatabase") when
        every plaintext is nil."""
        return _serialized_byte_count([self])

    def serialize(self) -> bytes:
        """ProcessedDatabase.serialize() (IndexPirProtocol.swift:360-378), packed on the device: the version byte, the
        little-endian UInt32 plaintext count, then per plaintext a tag (0 nil, 1 present) and its Eval rows."""
        return _serialize_databases([self]).tobytes()

    def save(self, path) -> None:
        """ProcessedDatabase.save(to:) (IndexPirProtocol.swift:350-355), written straight into the file's pages."""
        _save_databases([self], path)

    @staticmethod
    def load(context: Context, source, tableCount: int = 1) -> List["ProcessedDatabase"]:
        """ProcessedDatabase(from:context:) (IndexPirProtocol.swift:286-334) unpacked on the device, cut into
        `tableCount` databases of equal size (1 for index PIR; hashFunctionCount for a keyword-PIR shard,
        KeywordPirProtocol.swift:161-171).  source: bytes, a uint8 array, or a path, which is read through np.memmap so
        that a file larger than a host buffer streams.  Raises HeError with the reference's error name when the bytes are
        refused, and also where the reference would accept a residue >= its modulus or trap on a truncated buffer."""
        data = _source_bytes(source)
        handles = (C.c_void_p * max(1, tableCount))()
        buffer = data if data.size else np.zeros(1, dtype=np.uint8)  # an empty source still has an address
        _check(load_library().hecuda_pir_databases_create_serialized(context._h, _ptr(buffer), data.size, tableCount,
                                                                     handles))
        count = int.from_bytes(data[1:5].tobytes(), "little") // tableCount
        return [ProcessedDatabase._adopt(context, C.c_void_p(h), count) for h in handles[:tableCount]]

    def close(self):
        if getattr(self, "_h", None) is not None:
            load_library().hecuda_pir_database_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _source_bytes(source) -> np.ndarray:
    """The bytes of a serialized database as a uint8 array; a path is mapped, not read."""
    if isinstance(source, (str, os.PathLike)):
        return np.memmap(source, dtype=np.uint8, mode="r") if os.path.getsize(source) else np.zeros(0, dtype=np.uint8)
    if isinstance(source, (bytes, bytearray, memoryview)):
        return np.frombuffer(source, dtype=np.uint8)
    return np.ascontiguousarray(np.asarray(source, dtype=np.uint8)).reshape(-1)


def _handles(databases: Sequence[ProcessedDatabase]):
    return (C.c_void_p * len(databases))(*[db._h for db in databases])


def _serialized_byte_count(databases: Sequence[ProcessedDatabase]) -> int:
    size = C.c_uint64(0)
    _check(load_library().hecuda_pir_databases_serialized_byte_count(_handles(databases), len(databases), C.byref(size)))
    return size.value


def _serialize_into(databases: Sequence[ProcessedDatabase], out: np.ndarray) -> None:
    written = C.c_uint64(0)
    _check(load_library().hecuda_pir_databases_serialize(_handles(databases), len(databases), _ptr(out), out.size,
                                                         C.byref(written)))


def _serialize_databases(databases: Sequence[ProcessedDatabase]) -> np.ndarray:
    """The databases' plaintexts serialized as one ProcessedDatabase, in order (a keyword-PIR shard's layout)."""
    out = np.empty(_serialized_byte_count(databases), dtype=np.uint8)
    _serialize_into(databases, out)
    return out


def _save_databases(databases: Sequence[ProcessedDatabase], path) -> None:
    out = np.memmap(path, dtype=np.uint8, mode="w+", shape=(_serialized_byte_count(databases),))
    try:
        _serialize_into(databases, out)
        out.flush()
    except Exception:
        del out
        os.remove(path)
        raise


def _entry_arguments(database: Sequence[bytes], parameter: IndexPirParameter):
    """The entries as the C ABI takes them: concatenated bytes, entry_count + 1 offsets, and the dimensions."""
    if len(database) != parameter.entryCount:
        raise PirError(f"invalidDatabaseEntryCount(entryCount: {len(database)}, expected: {parameter.entryCount})")
    blobs = [bytes(e) for e in database]
    offsets = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    data = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)
    dims = (C.c_int32 * len(parameter.dimensions))(*parameter.dimensions)
    return data, offsets, dims


def packEntries(database: Sequence[bytes], context: Context, parameter: IndexPirParameter):
    """MulPirServer.plaintextRows on the device (hecuda_pir_process_entries): the coefficient rows (count x N) and the
    presence flags (count) of `process`, word for word."""
    data, offsets, dims = _entry_arguments(database, parameter)
    count = -(-parameter.encodedEntrySize // bytesPerPlaintext(context)) * int(np.prod(parameter.dimensions, dtype=np.int64))
    rows = np.empty((count, context.degree), dtype=np.uint64)
    present = np.empty(count, dtype=np.uint8)
    _check(load_library().hecuda_pir_process_entries(
        context._h, _ptr(data), _ptr(offsets), len(offsets) - 1, parameter.entrySizeInBytes,
        1 if parameter.encodingEntrySize else 0, dims, len(parameter.dimensions), _ptr(rows), _ptr(present), count))
    return rows, present


class PirWire:
    """Request / reply bytes of the index-PIR server (the payloads of the reference's protobuf messages)."""

    @staticmethod
    def computeResponse(server: "MulPirServer", queryPoly0, querySeeds, evaluationKey: EvaluationKey, indicesCount: int = 1):
        """Serialized seeded query ciphertexts in, serialized (skipLSBsForDecryption) reply ciphertexts out, one C-ABI call.
        queryPoly0: (count, byteCount(L rows)) uint8; querySeeds: (count, 32) uint8.  Returns (replies, skipLSBs) with
        replies of shape (indicesCount, chunkCount, bytes(poly0) + bytes(poly1))."""
        from . import Bfv
        ctx = server.context
        seeds = np.ascontiguousarray(np.asarray(querySeeds, dtype=np.uint8)).reshape(-1, 32)
        poly0 = np.ascontiguousarray(np.asarray(queryPoly0, dtype=np.uint8)).reshape(seeds.shape[0], -1)
        if poly0.shape[1] != Bfv.serializationByteCount(ctx, ctx.L):
            raise HeError(-1, "serializedBufferSizeMismatch")
        skips = skipLSBsForDecryption(ctx)
        sizes = [Bfv.serializationByteCount(ctx, 1, s) for s in skips]
        out = np.empty((indicesCount, server.chunkCount, sum(sizes)), dtype=np.uint8)
        handles = (C.c_void_p * len(server.databases))(*[db._h for db in server.databases])
        dims = (C.c_int32 * len(server.parameter.dimensions))(*server.parameter.dimensions)
        _check(load_library().hecuda_mulpir_compute_response_wire(
            ctx._h, evaluationKey._h, handles, len(server.databases), dims, len(server.parameter.dimensions), server.chunkCount,
            poly0.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p), seeds.shape[0], indicesCount, skips[0], skips[1],
            out.ctypes.data_as(C.c_void_p)))
        return out, skips

    @staticmethod
    def computeResponses(server: "MulPirServer", queryPoly0, querySeeds, evaluationKeys: Sequence[EvaluationKey],
                         indicesCount: int = 1):
        """computeResponse for many clients in one C-ABI call (hecuda_mulpir_compute_response_clients_wire): client c's
        serialized seeded query with evaluationKeys[c], its reply bytes identical to
        `computeResponse(server, queryPoly0[c], querySeeds[c], evaluationKeys[c], indicesCount)`.
        queryPoly0: (clients, count, byteCount(L rows)) uint8; querySeeds: (clients, count, 32) uint8.  Returns
        (replies, skipLSBs) with replies of shape (clients, indicesCount, chunkCount, bytes(poly0) + bytes(poly1))."""
        from . import Bfv
        ctx = server.context
        keys = list(evaluationKeys)
        seeds = np.ascontiguousarray(np.asarray(querySeeds, dtype=np.uint8))
        poly0 = np.ascontiguousarray(np.asarray(queryPoly0, dtype=np.uint8))
        size = Bfv.serializationByteCount(ctx, ctx.L)
        if not keys or seeds.size % (32 * len(keys)):
            raise HeError(-1, "serializedBufferSizeMismatch: querySeeds must be one set of 32-byte seeds per evaluation key")
        count = seeds.size // (32 * len(keys))
        if poly0.size != len(keys) * count * size:
            raise HeError(-1, f"serializedBufferSizeMismatch(poly0: {poly0.size} bytes, expected {len(keys) * count * size})")
        skips = skipLSBsForDecryption(ctx)
        sizes = [Bfv.serializationByteCount(ctx, 1, s) for s in skips]
        out = np.empty((len(keys), indicesCount, server.chunkCount, sum(sizes)), dtype=np.uint8)
        handles = (C.c_void_p * len(server.databases))(*[db._h for db in server.databases])
        key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
        dims = (C.c_int32 * len(server.parameter.dimensions))(*server.parameter.dimensions)
        _check(load_library().hecuda_mulpir_compute_response_clients_wire(
            ctx._h, key_handles, len(keys), handles, len(server.databases), dims, len(server.parameter.dimensions),
            server.chunkCount, poly0.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p), count, indicesCount,
            skips[0], skips[1], out.ctypes.data_as(C.c_void_p)))
        return out, skips


    @staticmethod
    def computeResponsesProto(server: "MulPirServer", messages: Sequence[bytes], evaluationKeys: Sequence[EvaluationKey],
                              indicesCount: int = 1) -> List[bytes]:
        """computeResponses with protobuf messages (hecuda_mulpir_compute_response_clients_proto): one
        pir.v1.EncryptedIndices per client in (num_pir_calls = indicesCount; its ciphertexts .seeded or .full), one
        api.pir.v1.PIRResponse per client out, whose reply ciphertexts hold the bytes computeResponses returns for the
        same poly0 and seeds.  The messages cross PCIe as they are; the replies are framed on the device."""
        ctx = server.context
        keys = list(evaluationKeys)
        buffers = [np.frombuffer(m, dtype=np.uint8) if isinstance(m, (bytes, bytearray, memoryview)) else
                   np.ascontiguousarray(m, dtype=np.uint8).reshape(-1) for m in messages]
        if not keys or len(buffers) != len(keys):
            raise HeError(-1, f"computeResponsesProto: {len(buffers)} messages for {len(keys)} evaluation keys")
        skips = skipLSBsForDecryption(ctx)
        size = C.c_uint64(0)
        _check(load_library().hecuda_mulpir_response_proto_byte_count(ctx._h, server.chunkCount, indicesCount, skips[0],
                                                                       skips[1], C.byref(size)))
        out = np.empty((len(keys), size.value), dtype=np.uint8)
        keep = [b if b.size else np.zeros(1, np.uint8) for b in buffers]
        counts = np.array([b.size for b in buffers], dtype=np.uint64)
        handles = (C.c_void_p * len(server.databases))(*[db._h for db in server.databases])
        key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
        dims = (C.c_int32 * len(server.parameter.dimensions))(*server.parameter.dimensions)
        _check(load_library().hecuda_mulpir_compute_response_clients_proto(
            ctx._h, key_handles, len(keys), handles, len(server.databases), dims, len(server.parameter.dimensions),
            server.chunkCount, (C.c_void_p * len(keep))(*[b.ctypes.data for b in keep]), counts.ctypes.data_as(C.c_void_p),
            indicesCount, skips[0], skips[1], out.ctypes.data_as(C.c_void_p)))
        return [row.tobytes() for row in out]


class PirRequestFields(C.Structure):
    """hecuda_pir_request_fields (include/hecuda.h)."""
    _fields_ = [("shard_index", C.c_uint32), ("has_shard_id", C.c_int32), ("has_query", C.c_int32),
                ("has_evaluation_key", C.c_int32), ("has_key_metadata", C.c_int32),
                ("shard_id_offset", C.c_uint64), ("shard_id_bytes", C.c_uint64),
                ("configuration_hash_offset", C.c_uint64), ("configuration_hash_bytes", C.c_uint64),
                ("query_offset", C.c_uint64), ("query_bytes", C.c_uint64),
                ("evaluation_key_offset", C.c_uint64), ("evaluation_key_bytes", C.c_uint64),
                ("key_timestamp", C.c_uint64), ("key_identifier_offset", C.c_uint64), ("key_identifier_bytes", C.c_uint64)]


class PirRequest:
    """api.pir.v1.PIRRequest, the envelope a PIR server receives."""

    @staticmethod
    def fields(data: bytes) -> dict:
        """The walk of a PIRRequest (hecuda_pir_request_fields_read), nothing copied on the host side: shardIndex,
        shardId (None when absent), configurationHash, the key metadata (keyTimestamp, keyIdentifier; from
        evaluation_key_metadata, or evaluation_key.metadata when that is absent) and the (offset, length) ranges of the
        query (an EncryptedIndices) and of evaluation_key.evaluation_key (a SerializedEvaluationKey), None when unset.
        Routing by shard and caching keys by identifier stay the caller's."""
        b = bytes(data)
        r = PirRequestFields()
        _check(load_library().hecuda_pir_request_fields_read(b, len(b), C.byref(r)))

        def span(offset, size):
            return b[offset:offset + size]

        return {
            "shardIndex": r.shard_index,
            "shardId": span(r.shard_id_offset, r.shard_id_bytes).decode() if r.has_shard_id else None,
            "configurationHash": span(r.configuration_hash_offset, r.configuration_hash_bytes),
            "keyTimestamp": r.key_timestamp if r.has_key_metadata else None,
            "keyIdentifier": span(r.key_identifier_offset, r.key_identifier_bytes) if r.has_key_metadata else None,
            "query": (r.query_offset, r.query_bytes) if r.has_query else None,
            "evaluationKey": (r.evaluation_key_offset, r.evaluation_key_bytes) if r.has_evaluation_key else None,
        }


class PirUtil:
    """enum PirUtil<Bfv<UInt64>> (PirUtil.swift:573): expansion and response computation on the device."""

    @staticmethod
    def expand(context: Context, ciphertexts, outputCount: int, evaluationKey: EvaluationKey) -> np.ndarray:
        cts = _host(ciphertexts)
        words = 2 * context.L * context.degree
        count = cts.size // words
        out = np.empty((outputCount, 2, context.L, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_mulpir_expand(context._h, evaluationKey._h, _ptr(cts), count, outputCount, _ptr(out)))
        return out


def _written(call) -> bytes:
    """A host-only writer's bytes: its size first, then the bytes."""
    written = C.c_uint64(0)
    _check(call(None, 0, C.byref(written)))
    out = np.empty(max(written.value, 1), dtype=np.uint8)
    _check(call(out.ctypes.data_as(C.c_void_p), out.size, C.byref(written)))
    return out[:written.value].tobytes()


def evaluationKeyMessage(context: Context, form) -> bytes:
    """SerializedEvaluationKey.proto() of a seeded key in EvaluationKey.generate(..., wire=True)'s form: the galois_key
    map in the form's element order, then the relinearization key (hecuda_pir_evaluation_key_write)."""
    arrays = EvaluationKey._wireArrays(context)
    relin = arrays(form["relinPoly0"], form["relinSeeds"]) if form.get("relinPoly0") is not None else None
    galois = {int(e): arrays(*v) for e, v in (form.get("galois") or {}).items()}
    elements = np.ascontiguousarray(list(galois), dtype=np.uint32)
    gp = np.ascontiguousarray(np.concatenate([v[0].reshape(-1) for v in galois.values()])) if galois else None
    gs = np.ascontiguousarray(np.concatenate([v[1].reshape(-1) for v in galois.values()])) if galois else None
    return _written(lambda out, capacity, written: load_library().hecuda_pir_evaluation_key_write(
        context._h, _ptr(relin[0]) if relin else None, _ptr(relin[1]) if relin else None,
        _ptr(elements) if galois else None, len(galois), _ptr(gp) if galois else None, _ptr(gs) if galois else None,
        out, capacity, written))


def responseFromMessage(context: Context, message: bytes, indicesCount: int, parameter) -> np.ndarray:
    """Response.native() of an api.pir.v1.PIRResponse: (indicesCount, chunkCount, 2, 1, N) Coeff ciphertexts, the
    replies found by hecuda_pir_response_read and their polys loaded with Bfv.skipLSBsForDecryption."""
    b = np.frombuffer(bytes(message), dtype=np.uint8)
    skips = skipLSBsForDecryption(context)
    sizes = [Bfv.serializationByteCount(context, 1, s) for s in skips]
    chunks = -(-parameter.encodedEntrySize // bytesPerPlaintext(context))  # MulPirServer.chunkCount
    offsets = np.empty(indicesCount * chunks, dtype=np.uint64)
    _check(load_library().hecuda_pir_response_read(context._h, b.ctypes.data_as(C.c_void_p), b.size, chunks, indicesCount,
                                                   skips[0], skips[1], offsets.ctypes.data_as(C.c_void_p)))
    polys = []
    for p, (skip, size) in enumerate(zip(skips, sizes)):
        start = offsets.astype(np.int64) + (sizes[0] if p else 0)
        rows = np.stack([b[o:o + size] for o in start])
        polys.append(Bfv.load(context, rows, 1, skip))
    return np.stack(polys, axis=1).reshape(indicesCount, chunks, 2, 1, context.degree)


class MulPirClient:
    """MulPirClient<PirUtil<Bfv<UInt64>>> (MulPir.swift:119-290): evaluation keys, queries and reply decryption, on the
    device."""

    def __init__(self, parameter: IndexPirParameter, context: Context):
        self.parameter, self.context = parameter, context

    @property
    def evaluationKeyConfig(self) -> EvaluationKeyConfig:
        return self.parameter.evaluationKeyConfig

    @property
    def entryChunksPerPlaintext(self) -> int:
        per_plaintext, encoded = bytesPerPlaintext(self.context), self.parameter.encodedEntrySize
        return per_plaintext // encoded if per_plaintext >= encoded else 1

    def generateEvaluationKey(self, secretKey: SecretKey) -> EvaluationKey:
        """MulPirClient.generateEvaluationKey (MulPir.swift:171-174)."""
        return EvaluationKey.generate(self.context, self.evaluationKeyConfig, secretKey)

    def computeCoordinates(self, index: int) -> List[int]:
        """MulPirClient.computeCoordinates (MulPir.swift:181-193)."""
        if not 0 <= index < self.parameter.entryCount:
            raise PirError(f"invalidIndex(index: {index}, numberOfEntries: {self.parameter.entryCount})")
        plaintext_index = index // self.entryChunksPerPlaintext
        product = int(np.prod(self.parameter.dimensions, dtype=np.int64))
        coordinates = []
        for size in self.parameter.dimensions:
            product //= size
            coordinate = plaintext_index // product
            plaintext_index -= coordinate * product
            coordinates.append(coordinate)
        return coordinates

    def generateQuery(self, indices: Sequence[int], secretKey: SecretKey) -> np.ndarray:
        """MulPirClient.generateQuery (MulPir.swift:201-218) with PirUtil.compressBinaryInputs (PirUtil.swift:361-404):
        Query.ciphertexts as (count, 2, L, N) Coeff."""
        return Bfv.encrypt(self.context, secretKey, self._queryPlaintexts(indices))

    def queryMessage(self, indices: Sequence[int], secretKey: SecretKey, aSeeds=None, errorSeeds=None) -> bytes:
        """generateQuery as the reference's client sends it: Query.proto(), a pir.v1.EncryptedIndices of .seeded
        ciphertexts with num_pir_calls = len(indices) (hecuda_pir_encrypted_indices_write)."""
        poly0, seeds = Bfv.encrypt(self.context, secretKey, self._queryPlaintexts(indices), seeded=True, aSeeds=aSeeds,
                                   errorSeeds=errorSeeds)
        return _written(lambda out, capacity, written: load_library().hecuda_pir_encrypted_indices_write(
            self.context._h, _ptr(poly0), _ptr(seeds), seeds.shape[0], len(indices), out, capacity, written))

    def evaluationKeyMessage(self, secretKey: SecretKey):
        """generateEvaluationKey as the reference's client sends it: (key, SerializedEvaluationKey.proto() bytes), the
        key's seeded form framed by hecuda_pir_evaluation_key_write."""
        key, form = EvaluationKey.generate(self.context, self.evaluationKeyConfig, secretKey, wire=True)
        return key, evaluationKeyMessage(self.context, form)

    def decryptResponseMessage(self, message: bytes, indices: Sequence[int], secretKey: SecretKey) -> List[bytes]:
        """decrypt of an api.pir.v1.PIRResponse: its reply ciphertexts found by hecuda_pir_response_read, their polys
        loaded with Bfv.skipLSBsForDecryption, then decrypt."""
        return self.decrypt(responseFromMessage(self.context, message, len(indices), self.parameter), indices, secretKey)

    def _queryPlaintexts(self, indices: Sequence[int]) -> np.ndarray:
        ctx, dims = self.context, self.parameter.dimensions
        accumulated, positions = 0, []
        for index in indices:
            coordinates = self.computeCoordinates(int(index))
            for dim, size in enumerate(dims):
                positions.append(accumulated + coordinates[dim])
                accumulated += size
        t, n = ctx.plaintextModulus, ctx.degree
        remaining, processed, plaintexts = self.parameter.expandedQueryCount * len(indices), 0, []
        while remaining > 0:
            count = min(remaining, n)
            raw = np.zeros(n, dtype=np.uint64)  # compressInputsForOneCiphertext: 2^-ceilLog2(count) mod t at the positions
            inverse = pow(pow(2, _ceil_log2(count), t), -1, t)
            for position in positions:
                if processed <= position < processed + count:
                    raw[position - processed] = inverse
            plaintexts.append(raw)
            processed += count
            remaining -= count
        return np.stack(plaintexts)

    def decryptFull(self, response, secretKey: SecretKey) -> List[bytes]:
        """MulPirClient.decryptFull: every reply's bytes.  response: (replies, chunkCount, 2, 1, N)."""
        ctx = self.context
        cts = _host(response)
        replies = cts.shape[0]
        plain = Bfv.decrypt(ctx, cts.reshape(-1, 2, cts.shape[-2], ctx.degree), secretKey).reshape(replies, -1, ctx.degree)
        bits = ctx.plaintextModulus.bit_length() - 1
        return [b"".join(CoefficientPacking.coefficientsToBytes(p, bits) for p in reply) for reply in plain]

    def decrypt(self, response, indices: Sequence[int], secretKey: SecretKey) -> List[bytes]:
        """MulPirClient.decrypt (MulPir.swift:245-275): decrypt, coefficient decode, bytes, the entry's range and its
        entry-size prefix."""
        cts = _host(response)
        if cts.shape[0] != len(indices):
            raise PirError(f"invalidResponse(replyCount: {cts.shape[0]}, expected: {len(indices)})")
        encoded, width = self.parameter.encodedEntrySize, self.parameter.entrySizeEncodingWidth
        out = []
        for data, index in zip(self.decryptFull(cts, secretKey), indices):
            position = int(index) % self.entryChunksPerPlaintext
            entry = data[position * encoded:(position + 1) * encoded]
            if self.parameter.encodingEntrySize:
                entry = entry[width:][:int.from_bytes(entry[:width], "little")]
            out.append(entry)
        return out

    def noiseBudget(self, response, secretKey: SecretKey) -> float:
        """Response.noiseBudget(using:variableTime:) (IndexPirProtocol.swift:742-747): the least budget of its ciphertexts.
        Must not be shared with another party."""
        cts = _host(response)
        if cts.size == 0:
            return -float("inf")
        return float(np.min(Bfv.noiseBudget(self.context, secretKey, cts.reshape(-1, 2, cts.shape[-2], self.context.degree))))


@dataclass
class ShardValidationResult:
    """ShardValidationResult (IndexPirProtocol.swift): the first trial's key and query, the last response, the least
    noise budget over the trials, each trial's response time (seconds) and entries per response."""

    evaluationKey: Any
    query: Any
    response: np.ndarray
    noiseBudget: float
    computeTimes: List[float]
    entryCountPerResponse: List[int]
    decryptedRow: Optional[bytes] = None  # the last trial's decrypted value (equal to the row's)


def _validate(trials: int, client, server_response, generate_query, decrypt, value: bytes, count_entries) -> ShardValidationResult:
    """The trial loop shared by the index and keyword validations (IndexPirProtocol.swift:420-484,
    KeywordDatabase.swift:557-630): a fresh secret key, evaluation key and query per trial, the response timed, its noise
    budget, and its decryption compared with the row."""
    if trials <= 0:
        raise PirError(f"Invalid trialsPerShard: {trials}")
    ctx = client.context
    first_key = first_query = response = None
    min_budget, times, counts = float("inf"), [], []
    for trial in range(trials):
        secret_key = SecretKey.generate(ctx)
        key = client.generateEvaluationKey(secret_key)
        query = generate_query(secret_key)
        start = time.perf_counter()
        response = server_response(query, key)
        times.append(time.perf_counter() - start)
        budget = client.noiseBudget(response, secret_key)
        min_budget = min(min_budget, budget)
        decrypted = decrypt(response, secret_key)
        if decrypted != value:
            if budget < Bfv.minNoiseBudget:
                raise PirError("Insufficient noise budget")
            raise PirError("Incorrect PIR response")
        counts.append(count_entries(response, secret_key))
        if trial == 0:
            first_key, first_query = key, query
        else:
            key.close()
    return ShardValidationResult(first_key, first_query, response, min_budget, times, counts, decrypted)


class MulPirServer:
    """MulPirServer<PirUtil<Bfv<UInt64>>> (MulPir.swift:292-426)."""

    def __init__(self, parameter: IndexPirParameter, context: Context, databases: Sequence[ProcessedDatabase]):
        self.parameter, self.context, self.databases = parameter, context, list(databases)
        expected = self.chunkCount * int(np.prod(parameter.dimensions, dtype=np.int64))
        for db in self.databases:
            if db.count != expected:
                raise PirError(f"invalidDatabasePlaintextCount(plaintextCount: {db.count}, expected: {expected})")

    @property
    def chunkCount(self) -> int:
        return -(-self.parameter.encodedEntrySize // bytesPerPlaintext(self.context))

    @staticmethod
    def load(path, parameter: IndexPirParameter, context: Context) -> "MulPirServer":
        """A server over the processed database saved at `path` (ProcessedDatabase(from:context:),
        IndexPirProtocol.swift:286-334); PirError("invalidDatabasePlaintextCount...") when it does not fit `parameter`."""
        databases = ProcessedDatabase.load(context, path)
        try:
            return MulPirServer(parameter, context, databases)
        except Exception:
            for db in databases:
                db.close()
            raise

    @staticmethod
    def process(database: Sequence[bytes], context: Context, parameter: IndexPirParameter) -> ProcessedDatabase:
        """MulPirServer.process (MulPir.swift:433-556): bytes -> coefficient plaintexts (host), Eval conversion (device)."""
        rows, present = MulPirServer.plaintextRows(database, context, parameter)
        return ProcessedDatabase(context, rows, present, evalFormat=False)

    @staticmethod
    def plaintextRows(database: Sequence[bytes], context, parameter: IndexPirParameter):
        """The host half of `process`: the coefficient vector of every plaintext slot, in database order, and which slots
        are non-nil.  `context` only needs `degree` and `plaintextModulus`."""
        if len(database) != parameter.entryCount:
            raise PirError(f"invalidDatabaseEntryCount(entryCount: {len(database)}, expected: {parameter.entryCount})")
        longest = max((len(e) for e in database), default=0)
        if longest > parameter.entrySizeInBytes:
            raise PirError(f"invalidDatabaseEntrySize(maximumEntrySize: {longest}, expected: {parameter.entrySizeInBytes})")
        capacity = bytesPerPlaintext(context)
        bits = context.plaintextModulus.bit_length() - 1
        encoded, width = parameter.encodedEntrySize, parameter.entrySizeEncodingWidth
        chunks = -(-encoded // capacity)
        per_chunk = int(np.prod(parameter.dimensions, dtype=np.int64))
        columns = per_chunk // parameter.dimensions[0]
        if chunks > 1:                                     # processSplitLargeEntries
            grid = [[None] * chunks for _ in range(per_chunk)]
            for row, entry in enumerate(database):
                entry = bytes(entry)
                blob = (len(entry).to_bytes(width, "little") if width else b"") + entry
                for chunk in range(chunks):
                    lo = chunk * capacity
                    # the reference cuts [lo - width, lo - width + capacity) out of the entry, prefixing the size to chunk 0
                    hi = min(lo - width + capacity, len(entry)) + width
                    if lo - width < hi - width:
                        grid[row][chunk] = blob[lo:hi] if chunk else blob[:hi]
            order = [(row, chunk) for chunk in range(chunks) for skip in range(columns)
                     for row in range(skip, per_chunk, columns)]
            pieces = [grid[row][chunk] for row, chunk in order]
        else:                                              # processPackEntries
            stride = (capacity // encoded) * encoded
            flat = bytearray()
            for entry in database:
                entry = bytes(entry)
                body = (len(entry).to_bytes(width, "little") if width else b"") + entry
                flat += body.ljust(encoded, b"\0")
            packed = [bytes(flat[i:i + stride]) for i in range(0, len(flat), stride)]
            packed += [None] * (per_chunk - len(packed))
            pieces = [packed[row] for skip in range(columns) for row in range(skip, per_chunk, columns)]
        return _pack_rows(pieces, bits, context.degree)

    @staticmethod
    def processOnDevice(database: Sequence[bytes], context: Context, parameter: IndexPirParameter) -> ProcessedDatabase:
        """MulPirServer.process (MulPir.swift:433-556) with the packing on the device as well
        (hecuda_pir_database_create_from_entries): only the entry bytes cross PCIe.  The resident words equal those of
        `process(database, context, parameter)`."""
        data, offsets, dims = _entry_arguments(database, parameter)
        h = C.c_void_p()
        _check(load_library().hecuda_pir_database_create_from_entries(
            context._h, _ptr(data), _ptr(offsets), len(offsets) - 1, parameter.entrySizeInBytes,
            1 if parameter.encodingEntrySize else 0, dims, len(parameter.dimensions), C.byref(h)))
        count = -(-parameter.encodedEntrySize // bytesPerPlaintext(context)) * int(np.prod(parameter.dimensions, dtype=np.int64))
        return ProcessedDatabase._adopt(context, h, count)

    def computeResponse(self, query, evaluationKey: EvaluationKey, indicesCount: int = 1) -> np.ndarray:
        """computeResponse(to:using:) -> Response.ciphertexts as (indicesCount, chunkCount, 2, 1, N) (Coeff, modulus q_0).

        query: Query.ciphertexts stacked, (queryCiphertextCount, 2, L, N) Coeff."""
        ctx = self.context
        cts = _host(query)
        words = 2 * ctx.L * ctx.degree
        if cts.size % words:
            raise HeError(-1, "invalidCiphertext: query must be ciphertexts of 2 x L x N")
        handles = (C.c_void_p * len(self.databases))(*[db._h for db in self.databases])
        dims = (C.c_int32 * len(self.parameter.dimensions))(*self.parameter.dimensions)
        out = np.empty((indicesCount, self.chunkCount, 2, 1, ctx.degree), dtype=np.uint64)
        _check(load_library().hecuda_mulpir_compute_response(
            ctx._h, evaluationKey._h, handles, len(self.databases), dims, len(self.parameter.dimensions), self.chunkCount,
            _ptr(cts), cts.size // words, indicesCount, _ptr(out)))
        return out

    def computeResponses(self, queries, evaluationKeys: Sequence[EvaluationKey], indicesCount: int = 1) -> np.ndarray:
        """computeResponse for many clients in one C-ABI call: client c's query with evaluationKeys[c], each reply
        bit-identical to `computeResponse(queries[c], evaluationKeys[c], indicesCount)`.  Groups of up to
        HECUDA_MULPIR_CLIENT_GROUP clients share one pass over each database.

        queries: (clients, queryCiphertextCount, 2, L, N) Coeff.  Returns (clients, indicesCount, chunkCount, 2, 1, N)."""
        ctx = self.context
        keys = list(evaluationKeys)
        cts = _host(queries)
        words = 2 * ctx.L * ctx.degree
        if not keys or cts.size % (words * len(keys)):
            raise HeError(-1, "invalidCiphertext: queries must be one set of 2 x L x N ciphertexts per evaluation key")
        handles = (C.c_void_p * len(self.databases))(*[db._h for db in self.databases])
        key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
        dims = (C.c_int32 * len(self.parameter.dimensions))(*self.parameter.dimensions)
        out = np.empty((len(keys), indicesCount, self.chunkCount, 2, 1, ctx.degree), dtype=np.uint64)
        _check(load_library().hecuda_mulpir_compute_response_clients(
            ctx._h, key_handles, len(keys), handles, len(self.databases), dims, len(self.parameter.dimensions),
            self.chunkCount, _ptr(cts), cts.size // (words * len(keys)), indicesCount, _ptr(out)))
        return out

    def validate(self, row: Tuple[int, bytes], trials: int = 1) -> ShardValidationResult:
        """ProcessedDatabaseWithParameters.validate(row:trials:) (IndexPirProtocol.swift:420-484) against the first
        database: row = (index, value).  Every step runs on the device; raises PirError("Insufficient noise budget") or
        PirError("Incorrect PIR response") when a trial's reply does not decrypt to the value."""
        index, value = int(row[0]), bytes(row[1])
        client = MulPirClient(self.parameter, self.context)
        return _validate(trials, client, lambda query, key: self.computeResponse(query, key),
                         lambda sk: client.generateQuery([index], sk),
                         lambda response, sk: client.decrypt(response, [index], sk)[0], value, lambda response, sk: 1)
