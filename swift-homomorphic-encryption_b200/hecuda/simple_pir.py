"""hecuda.simple_pir -- the reference's SimplePIR server over libhecuda.

Names follow Sources/PrivateInformationRetrieval/SimplePir/:

    SimplePirEncryptionParams, SimplePirParameters          SimplePir.swift:19-160
    SimplePirServer.computingParams / process               SimplePir+Database.swift:208-290
    SimplePirServer(processedDatabase:hint:params:)         SimplePir+Server.swift:24-29
    SimplePirServer.computeResponse                         SimplePir+Server.swift:31-38
    Array2d.save / init(from:)                              SimplePir+Database.swift:36-121
    DatabaseMap, DatabaseMap.shardDatabase                  SimplePir/DatabaseMap.swift:18-110
    ShardMap                                                SimplePir/SimplePir+Shards.swift:18-45
    DefaultQueryGenerator, PrecomputedQueries               SimplePir/SimplePir+Precompute.swift:191-356
    SimplePirClient                                         SimplePir/SimplePir+Client.swift:98-127
    SimplePirClientForAllShards                             SimplePir/SimplePir+Shards.swift:47-173
    SimplePirServer.validate / SimplePirShardedServer.validate   verifyProcessing, SimplePIRProcessDatabase/main.swift:260-348
    SimplePIRProcessDatabase's sharding and file names      Sources/SimplePIRProcessDatabase/main.swift:158-253
    SimplePIRRequest / SimplePIRResponse / SimplePIRConfig  ApplicationProtobuf/PirConversion.swift:380-518,
                                                            api/pir/v1/pir.proto, SimplePIRProcessDatabase/main.swift:193-258

The processed database stays on the device as u8 digit planes; responses are integer tensor-core products there.
`scalar` is the reference's Scalar type: np.uint32 (UInt32) or np.uint64 (UInt64).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import secrets
import struct
import time
from collections import deque
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _MAX_LOG2_Q_STDDEV32, _MAX_LOG2_Q_STDDEV64, _check, _ptr, load_library
from .pir import PirError

SEED_BYTES = 32  # NistAes128Ctr.SeedCount



class _Params(C.Structure):  # hecuda_simple_pir_params
    _fields_ = [("plaintext_modulus_bits", C.c_int32), ("ciphertext_modulus_bits", C.c_int32),
                ("lattice_dimension", C.c_int64), ("entry_size", C.c_int64), ("entries_per_column", C.c_int64),
                ("chunks_per_entry", C.c_int64), ("database_columns", C.c_int64), ("word_bits", C.c_int32),
                ("error_std_dev", C.c_double)]


@dataclass(frozen=True)
class SimplePirEncryptionParams:
    """errorStdDev is 3.2 (.stdDev32) or 6.4 (.stdDev64); securityLevel "quantum128" or "unchecked"."""
    plaintextModulusBits: int
    ciphertextModulusBits: int
    latticeDimension: int
    errorStdDev: float = 3.2
    securityLevel: str = "quantum128"

    def __post_init__(self):
        n = self.latticeDimension
        if n < 1 or n & (n - 1):
            raise PirError(f"invalidEncryptionParameters: SimplePir latticeDimension={n} is not a power of 2")
        if self.errorStdDev not in (3.2, 6.4):
            raise PirError(f"invalidEncryptionParameters: errorStdDev must be 3.2 (.stdDev32) or 6.4 (.stdDev64), "
                           f"got {self.errorStdDev}")
        if self.ciphertextModulusBits <= self.plaintextModulusBits:
            raise PirError("invalidEncryptionParameters: SimplePir ciphertextModulusBits must be > plaintextModulusBits")
        if self.securityLevel == "unchecked":
            return
        table = _MAX_LOG2_Q_STDDEV64 if self.errorStdDev == 6.4 else _MAX_LOG2_Q_STDDEV32
        if n not in table:
            raise PirError(f"invalidEncryptionParameters: no quantum128 bound for latticeDimension={n}, "
                           f"errorStdDev={self.errorStdDev}")
        if self.ciphertextModulusBits > table[n]:
            raise PirError(f"insecureEncryptionParameters: ciphertextModulusBits={self.ciphertextModulusBits} "
                           f"exceeds {table[n]} for latticeDimension={n}")


def _coeff_count(byte_count: int, bits: int) -> int:  # CoefficientPacking.bytesToCoefficientsCoeffCount(decode: false)
    return -(-byte_count * 8 // bits)


@dataclass(frozen=True)
class SimplePirParameters:
    encryptionParams: SimplePirEncryptionParams
    entrySizeInBytes: int
    entriesPerColumn: int
    chunksPerEntry: int
    databaseColumns: int
    seed: bytes = field(default=b"\0" * SEED_BYTES)

    def __post_init__(self):
        if not (self.entriesPerColumn == 1 or self.chunksPerEntry == 1):
            raise PirError("SimplePirParameters: entriesPerColumn == 1 || chunksPerEntry == 1")

    plaintextModulusBits = property(lambda self: self.encryptionParams.plaintextModulusBits)
    ciphertextModulusBits = property(lambda self: self.encryptionParams.ciphertextModulusBits)
    latticeDimension = property(lambda self: self.encryptionParams.latticeDimension)

    @property
    def entrySizeInScalar(self) -> int:
        return _coeff_count(self.entrySizeInBytes, self.plaintextModulusBits)

    @property
    def chunkSize(self) -> int:
        return -(-self.entrySizeInScalar // self.chunksPerEntry)

    @property
    def columnSize(self) -> int:
        return self.entriesPerColumn * self.entrySizeInScalar if self.chunksPerEntry == 1 else self.chunkSize

    @property
    def aPolyCount(self) -> int:
        return -(-self.databaseColumns // self.latticeDimension)

    @staticmethod
    def computingParams(encryptionParams: SimplePirEncryptionParams, entryCount: int, entrySizeInBytes: int,
                        seed: Optional[bytes] = None) -> "SimplePirParameters":
        """SimplePirServerProtocol.computingParams (SimplePir+Database.swift:208-243).  Swift's .rounded() rounds halves
        away from zero (floor(x + 0.5) here, every operand being >= 0), and chunksPerEntry truncates."""
        scalars = _coeff_count(entrySizeInBytes, encryptionParams.plaintextModulusBits)
        ideal_column = min(math.floor(math.sqrt(float(entryCount * scalars)) + 0.5), scalars)
        entries_per_column = max(math.floor(float(ideal_column) / float(scalars) + 0.5), 1)
        chunks_per_entry = max(int(float(scalars) / float(ideal_column)), 1)
        columns = entryCount * chunks_per_entry if entries_per_column == 1 else max(-(-entryCount // entries_per_column), 1)
        return SimplePirParameters(encryptionParams, entrySizeInBytes, entries_per_column, chunks_per_entry, columns,
                                   secrets.token_bytes(SEED_BYTES) if seed is None else bytes(seed))

    def _c(self, word_bits: int) -> _Params:
        return _Params(self.plaintextModulusBits, self.ciphertextModulusBits, self.latticeDimension, self.entrySizeInBytes,
                       self.entriesPerColumn, self.chunksPerEntry, self.databaseColumns, word_bits,
                       self.encryptionParams.errorStdDev)


def _word_bits(scalar) -> int:
    scalar = np.dtype(scalar)
    if scalar not in (np.dtype(np.uint32), np.dtype(np.uint64)):
        raise PirError("SimplePir scalar must be np.uint32 or np.uint64")
    return scalar.itemsize * 8


def save_array2d(array: np.ndarray, path: str):
    """Array2d.save(to:): u32 LE row and column counts, then the scalars little-endian."""
    array = np.asarray(array)
    with open(path, "wb") as f:
        f.write(struct.pack("<II", array.shape[0], array.shape[1]))
        f.write(np.ascontiguousarray(array, dtype=array.dtype.newbyteorder("<")).tobytes())


def load_array2d(path: str, scalar=np.uint64) -> np.ndarray:
    """Array2d(from:); PirError.corruptedData on a truncated file."""
    dtype = np.dtype(scalar).newbyteorder("<")
    with open(path, "rb") as f:
        header = f.read(8)
        if len(header) < 8:
            raise PirError("corruptedData: Unexpected EOF")
        rows, cols = struct.unpack("<II", header)
        if rows * cols >= 16_000_000_000:
            raise PirError(f"corruptedData: Database is unreasonably large: {rows} x {cols}")
        body = f.read(rows * cols * dtype.itemsize)
    if len(body) < rows * cols * dtype.itemsize:
        raise PirError("corruptedData: Unexpected EOF")
    return np.frombuffer(body, dtype=dtype).astype(np.dtype(scalar)).reshape(rows, cols)


class SimplePirDatabase:
    """The processed database (columnSize x databaseColumns), resident on the device."""

    def __init__(self, handle, params: SimplePirParameters, scalar):
        self._h, self.params, self.scalar = handle, params, np.dtype(scalar)

    @staticmethod
    def create(processedDatabase, params: SimplePirParameters, scalar=np.uint64) -> "SimplePirDatabase":
        bits = _word_bits(scalar)
        matrix = np.ascontiguousarray(np.asarray(processedDatabase, dtype=scalar))
        if matrix.shape != (params.columnSize, params.databaseColumns):
            raise PirError(f"processed database must be {params.columnSize} x {params.databaseColumns}, got {matrix.shape}")
        h = C.c_void_p()
        cp = params._c(bits)
        _check(load_library().hecuda_simple_pir_database_create(_ptr(matrix), C.byref(cp), C.byref(h)))
        return SimplePirDatabase(h, params, scalar)

    def export(self) -> np.ndarray:
        out = np.empty((self.params.columnSize, self.params.databaseColumns), dtype=self.scalar)
        _check(load_library().hecuda_simple_pir_database_export(self._h, _ptr(out)))
        return out

    def save(self, path: str):
        save_array2d(self.export(), path)

    @staticmethod
    def load(path: str, params: SimplePirParameters, scalar=np.uint64) -> "SimplePirDatabase":
        return SimplePirDatabase.create(load_array2d(path, scalar), params, scalar)

    def close(self):
        if self._h is not None:
            load_library().hecuda_simple_pir_database_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class SimplePIRProcessDatabaseResults:
    database: SimplePirDatabase
    hint: np.ndarray
    params: SimplePirParameters


class SimplePirServer:
    """SimplePirServer<Scalar>: construct from a processed database (host matrix or SimplePirDatabase), its hint and
    params; SimplePirServer.process builds all three from raw entries on the device."""

    def __init__(self, processedDatabase, hint, params: SimplePirParameters, scalar=np.uint64):
        self.scalar = np.dtype(scalar)
        _word_bits(self.scalar)
        self.database = (processedDatabase if isinstance(processedDatabase, SimplePirDatabase)
                         else SimplePirDatabase.create(processedDatabase, params, self.scalar))
        self.hint = np.asarray(hint, dtype=self.scalar)
        self.params = params

    @staticmethod
    def process(database, encryptionParams: SimplePirEncryptionParams, seed: Optional[bytes] = None,
                scalar=np.uint64) -> SimplePIRProcessDatabaseResults:
        """database: entryCount x entrySizeInBytes uint8 (RawDatabase = Array2d<UInt8>)."""
        bits = _word_bits(scalar)
        raw = np.ascontiguousarray(np.asarray(database, dtype=np.uint8))
        if raw.ndim != 2 or raw.shape[0] < 1 or raw.shape[1] < 1:
            raise PirError("SimplePir database must be a non-empty entryCount x entrySizeInBytes byte matrix")
        params = SimplePirParameters.computingParams(encryptionParams, raw.shape[0], raw.shape[1], seed)
        if len(params.seed) != SEED_BYTES:
            raise PirError(f"seed must be {SEED_BYTES} bytes")
        hint = np.empty((params.columnSize, params.latticeDimension), dtype=scalar)
        seed_buf = np.frombuffer(params.seed, dtype=np.uint8).copy()
        h = C.c_void_p()
        cp = params._c(bits)
        _check(load_library().hecuda_simple_pir_process(_ptr(raw), raw.shape[0], C.byref(cp), _ptr(seed_buf), _ptr(hint),
                                                        C.byref(h)))
        return SimplePIRProcessDatabaseResults(SimplePirDatabase(h, params, scalar), hint, params)

    def _requests(self, requests) -> np.ndarray:
        r = np.ascontiguousarray(np.asarray(requests, dtype=self.scalar))
        if r.ndim == 2:
            r = r[None]
        if r.ndim != 3 or r.shape[1:] != (self.params.chunksPerEntry, self.params.databaseColumns):
            raise PirError(f"request must be {self.params.chunksPerEntry} x {self.params.databaseColumns}, got "
                           f"{np.asarray(requests).shape}")
        return r

    def computeResponses(self, requests: Sequence) -> np.ndarray:
        """Responses to many requests in one device pass: count x chunksPerEntry x columnSize."""
        r = self._requests(np.stack([np.asarray(x, dtype=self.scalar) for x in requests]) if isinstance(requests, list)
                           else requests)
        out = np.empty((r.shape[0], self.params.chunksPerEntry, self.params.columnSize), dtype=self.scalar)
        _check(load_library().hecuda_simple_pir_compute_response(self.database._h, _ptr(r), r.shape[0], _ptr(out)))
        return out

    def computeResponse(self, requests) -> np.ndarray:
        """computeResponse(to:): chunksPerEntry x K request words -> chunksPerEntry x columnSize."""
        return self.computeResponses(self._requests(requests))[0]

    def computeResponsesDevice(self, requests_ptr: int, count: int, responses_ptr: int, stream: int = 0):
        """Device buffers (torch data_ptr()): enqueue on `stream` without synchronising."""
        _check(load_library().hecuda_simple_pir_compute_response_device(self.database._h, C.c_void_p(requests_ptr), count,
                                                                        C.c_void_p(responses_ptr), C.c_void_p(stream)))

    def computeResponsesProto(self, messages) -> list:
        """One SimplePIRResponse (bytes) per SimplePIRRequest (bytes, shard_index 0), in one device call."""
        return _responses_proto(_handles([self.database]), 1, messages)


# ---- sharding (DatabaseMap.swift, SimplePir+Shards.swift, SimplePIRProcessDatabase/main.swift:158-253)
@dataclass(frozen=True)
class ChunkLocation:
    shardIndex: int
    index: int


@dataclass(frozen=True)
class DatabaseMapEntry:  # DatabaseMap.Entry
    originalIndex: int
    size: int
    chunks: tuple


def _raw_entries(entries):
    """(originalIndex, bytes) pairs or an entryCount x entrySize uint8 matrix -> (original indices, values, uint64
    offsets with entryCount + 1 elements)."""
    if isinstance(entries, np.ndarray):
        raw = np.ascontiguousarray(entries, dtype=np.uint8)
        if raw.ndim != 2:
            raise PirError("entries must be a 2-D uint8 array or (originalIndex, bytes) pairs")
        count, size = raw.shape
        return (np.arange(count, dtype=np.int64), raw.reshape(-1),
                np.arange(count + 1, dtype=np.uint64) * np.uint64(size))
    pairs = list(entries)
    index = np.array([int(i) for i, _ in pairs], dtype=np.int64)
    values = [np.frombuffer(bytes(v), dtype=np.uint8) for _, v in pairs]
    offsets = np.zeros(len(values) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(v) for v in values], dtype=np.uint64)
    flat = np.concatenate(values) if values else np.zeros(0, dtype=np.uint8)
    return index, flat, offsets


def _chunk_locations(sizes: np.ndarray, shard_count: int, chunk_size: int, rng) -> np.ndarray:
    """shardDatabase's placement, vectorised: each entry draws its own permutation of the shards (one row of
    rng.permuted), chunk c goes to shard perm[c % shardCount] at the next free row.  -> chunks x 2 int64, entry-major."""
    counts = (sizes.astype(np.int64) + chunk_size - 1) // chunk_size
    perms = rng.permuted(np.tile(np.arange(shard_count, dtype=np.int64), (len(sizes), 1)), axis=1)
    entry = np.repeat(np.arange(len(sizes)), counts)
    chunk = np.arange(int(counts.sum())) - np.repeat(np.cumsum(counts) - counts, counts)
    shard = perms[entry, chunk % shard_count] if len(entry) else np.zeros(0, dtype=np.int64)
    order = np.argsort(shard, kind="stable")  # rows of a shard in entry-major order
    first = np.searchsorted(shard[order], np.arange(shard_count))
    index = np.empty_like(shard)
    index[order] = np.arange(len(shard)) - first[shard[order]]
    return np.ascontiguousarray(np.stack([shard, index], axis=1), dtype=np.int64)


class DatabaseMap:
    """DatabaseMap: entries (originalIndex, size, chunks of ChunkLocation(shardIndex, index)) and chunkSize.  The
    chunk locations are kept as one chunks x 2 array (entry-major); `entries` builds the reference's view of them."""

    def __init__(self, originalIndices, sizes, locations, chunkSize: int):
        self.originalIndices = np.asarray(originalIndices, dtype=np.int64)
        self.sizes = np.asarray(sizes, dtype=np.int64)
        self.chunkLocations = np.ascontiguousarray(locations, dtype=np.int64).reshape(-1, 2)
        self.chunkSize = chunkSize

    @property
    def entries(self) -> tuple:
        bounds = np.concatenate([[0], np.cumsum((self.sizes + self.chunkSize - 1) // self.chunkSize)])
        locs = [ChunkLocation(int(s), int(i)) for s, i in self.chunkLocations]
        return tuple(DatabaseMapEntry(int(self.originalIndices[e]), int(self.sizes[e]), tuple(locs[bounds[e]:bounds[e + 1]]))
                     for e in range(len(self.sizes)))

    def __eq__(self, other):
        return (isinstance(other, DatabaseMap) and self.chunkSize == other.chunkSize and
                np.array_equal(self.originalIndices, other.originalIndices) and np.array_equal(self.sizes, other.sizes)
                and np.array_equal(self.chunkLocations, other.chunkLocations))

    @staticmethod
    def shardDatabase(entries, shardCount: int, chunkSize: int, rng=None):
        """DatabaseMap.shardDatabase(entries:shardCount:chunkSize:) on the host -> (databaseMap, shards), each shard a
        rows x chunkSize uint8 matrix.  rng (numpy Generator) draws the permutations; the reference's draws from
        SystemRandomNumberGenerator cannot be reproduced."""
        if shardCount < 1 or chunkSize < 1:
            raise PirError("shardCount and chunkSize must be positive")
        index, values, offsets = _raw_entries(entries)
        sizes = np.diff(offsets).astype(np.int64)
        locations = _chunk_locations(sizes, shardCount, chunkSize, rng or np.random.default_rng())
        rows = np.bincount(locations[:, 0], minlength=shardCount)
        shards = [np.zeros((int(r), chunkSize), dtype=np.uint8) for r in rows]
        if len(sizes) and np.all(sizes == sizes[0]):  # equal sizes: every entry's zero-padded chunks at once
            per = -(-int(sizes[0]) // chunkSize)
            padded = np.zeros((len(sizes), per * chunkSize), dtype=np.uint8)
            padded[:, :sizes[0]] = values.reshape(len(sizes), -1)
            chunks = padded.reshape(-1, chunkSize)
            for s in range(shardCount):
                mine = locations[:, 0] == s
                shards[s][locations[mine, 1]] = chunks[mine]
        else:
            chunk = 0
            for e in range(len(sizes)):
                start = int(offsets[e])
                for c in range(0, int(sizes[e]), chunkSize):
                    s, i = locations[chunk]
                    piece = values[start + c:start + min(c + chunkSize, int(sizes[e]))]
                    shards[s][i, :len(piece)] = piece
                    chunk += 1
        return DatabaseMap(index, sizes, locations, chunkSize), shards


class ShardMap:
    """ShardMap(databaseMap:): shardCount counts the shards that hold a chunk; chunksPerShard = ceil(maximumChunkCount
    / shardCount)."""

    def __init__(self, databaseMap: DatabaseMap):
        self.mapping = {e.originalIndex: e for e in databaseMap.entries}
        self.shardCount = len({c.shardIndex for e in self.mapping.values() for c in e.chunks})
        self.maximumChunkCount = max((len(e.chunks) for e in self.mapping.values()), default=0)
        self.chunkSize = databaseMap.chunkSize
        self.chunksPerShard = -(-self.maximumChunkCount // self.shardCount) if self.shardCount else 0

    def __getitem__(self, originalIndex: int) -> Optional[DatabaseMapEntry]:
        return self.mapping.get(originalIndex)


def _handles(databases) -> C.Array:
    return (C.c_void_p * len(databases))(*[d._h.value if isinstance(d._h, C.c_void_p) else d._h for d in databases])


class SimplePirShardedServer:
    """One SimplePirServer per shard, answered together: computeResponses sends every client's requests to every shard
    in one grouped device pass.  process shards and processes raw entries on the device, as the
    SimplePIRProcessDatabase tool does."""

    def __init__(self, databases: Sequence[SimplePirDatabase], hints: Sequence[np.ndarray],
                 params: Sequence[SimplePirParameters], scalar=np.uint64, databaseMap: Optional[DatabaseMap] = None):
        self.scalar = np.dtype(scalar)
        _word_bits(self.scalar)
        if not (len(databases) == len(hints) == len(params)) or not databases:
            raise PirError("one database, hint and params per shard")
        self.databases, self.hints, self.params = list(databases), list(hints), list(params)
        self.databaseMap = databaseMap
        self._h = _handles(self.databases)

    @property
    def shardCount(self) -> int:
        return len(self.databases)

    @staticmethod
    def process(entries, encryptionParams: SimplePirEncryptionParams, shardCount: int, chunkSize: Optional[int] = None,
                seed: Optional[bytes] = None, scalar=np.uint64, rng=None) -> "SimplePirShardedServer":
        """entries: (originalIndex, bytes) pairs or an entryCount x entrySize uint8 matrix.  chunkSize None is the
        tool's ceil(largest entry / shardCount); seed None draws one seed per shard, given bytes seed every shard."""
        bits = _word_bits(scalar)
        if shardCount < 1:
            raise PirError("shardCount must be positive")
        index, values, offsets = _raw_entries(entries)
        sizes = np.diff(offsets).astype(np.int64)
        if chunkSize is None:
            chunkSize = -(-int(sizes.max(initial=0)) // shardCount)
        if chunkSize < 1:
            raise PirError("chunkSize must be positive")
        locations = _chunk_locations(sizes, shardCount, chunkSize, rng or np.random.default_rng())
        rows = np.bincount(locations[:, 0], minlength=shardCount)
        if seed is not None and len(seed) != SEED_BYTES:
            raise PirError(f"seed must be {SEED_BYTES} bytes")
        params = [SimplePirParameters.computingParams(encryptionParams, max(int(r), 1), chunkSize, seed) for r in rows]
        hints = [np.empty((p.columnSize, p.latticeDimension), dtype=scalar) for p in params]
        hint_buf = np.empty(sum(h.size for h in hints), dtype=scalar)
        seeds = np.frombuffer(b"".join(p.seed for p in params), dtype=np.uint8).copy()
        cparams = (_Params * shardCount)(*[p._c(bits) for p in params])
        handles = (C.c_void_p * shardCount)()
        values = values if values.size else np.zeros(1, dtype=np.uint8)
        _check(load_library().hecuda_simple_pir_process_shards(
            _ptr(values), _ptr(offsets), len(sizes), chunkSize, shardCount, _ptr(locations),
            cparams, _ptr(seeds), _ptr(hint_buf), handles))
        at = 0
        for h in hints:
            h[...] = hint_buf[at:at + h.size].reshape(h.shape)
            at += h.size
        databases = [SimplePirDatabase(C.c_void_p(handles[i]), params[i], scalar) for i in range(shardCount)]
        return SimplePirShardedServer(databases, hints, params, scalar, DatabaseMap(index, sizes, locations, chunkSize))

    def _words(self, requests_per_shard: int):
        inw = [requests_per_shard * p.chunksPerEntry * p.databaseColumns for p in self.params]
        outw = [requests_per_shard * p.chunksPerEntry * p.columnSize for p in self.params]
        return inw, outw

    def computeResponses(self, requests, requests_per_shard: Optional[int] = None):
        """requests: one entry per client, each a list of shardCount arrays requests_per_shard x chunksPerEntry_s x K_s
        (SimplePirClientForAllShards.query, flattened) -> the same nesting with columnSize_s in place of K_s.  A 2-D
        array count x words (client-major blocks) with requests_per_shard given returns count x response words."""
        flat = isinstance(requests, np.ndarray)
        if flat:
            if requests_per_shard is None:
                raise PirError("a flat request array needs requests_per_shard")
            r = np.ascontiguousarray(requests, dtype=self.scalar)
        else:
            requests = list(requests)
            if not requests:
                return []
            requests_per_shard = len(requests[0][0])
            blocks = []
            for client in requests:
                if len(client) != self.shardCount:
                    raise PirError(f"a client must send requests to all {self.shardCount} shards")
                for s, (q, p) in enumerate(zip(client, self.params)):
                    q = np.asarray(q, dtype=self.scalar)
                    if q.shape != (requests_per_shard, p.chunksPerEntry, p.databaseColumns):
                        raise PirError(f"shard {s}: requests must be {requests_per_shard} x {p.chunksPerEntry} x "
                                       f"{p.databaseColumns}, got {q.shape}")
                    blocks.append(q.reshape(-1))
            r = np.concatenate(blocks).reshape(len(requests), -1)
        inw, outw = self._words(requests_per_shard)
        if r.ndim != 2 or r.shape[1] != sum(inw):
            raise PirError(f"requests must be count x {sum(inw)} words")
        out = np.empty((r.shape[0], sum(outw)), dtype=self.scalar)
        _check(load_library().hecuda_simple_pir_compute_response_shards(self._h, self.shardCount, requests_per_shard,
                                                                        _ptr(r), r.shape[0], _ptr(out)))
        if flat:
            return out
        bounds = np.concatenate([[0], np.cumsum(outw)])
        return [[out[c, bounds[s]:bounds[s + 1]].reshape(requests_per_shard, p.chunksPerEntry, p.columnSize)
                 for s, p in enumerate(self.params)] for c in range(out.shape[0])]

    def computeResponsesDevice(self, requests_ptr: int, requests_per_shard: int, count: int, responses_ptr: int,
                               stream: int = 0):
        """Device buffers in the flat client-major layout: enqueue on `stream` without synchronising."""
        _check(load_library().hecuda_simple_pir_compute_response_shards_device(
            self._h, self.shardCount, requests_per_shard, C.c_void_p(requests_ptr), count, C.c_void_p(responses_ptr),
            C.c_void_p(stream)))

    def save(self, prefix: str, configPath: Optional[str] = None):
        """The tool's files: prefix-i.bin (processed database) and prefix-i.hint.bin for every shard i; with configPath,
        also the SimplePIRConfig (the databaseMap, every shard's params and the SHA-256 of every hint file,
        main.swift:231-258)."""
        for i, (db, hint) in enumerate(zip(self.databases, self.hints)):
            db.save(f"{prefix}-{i}.bin")
            save_array2d(hint, f"{prefix}-{i}.hint.bin")
        if configPath is not None:
            if self.databaseMap is None:
                raise PirError("the config needs the databaseMap")
            ids = []
            for i in range(self.shardCount):
                with open(f"{prefix}-{i}.hint.bin", "rb") as f:
                    ids.append(hashlib.sha256(f.read()).digest())
            SimplePirConfig(self.databaseMap, self.params, ids).save(configPath)

    @staticmethod
    def fromConfig(prefix: str, config) -> "SimplePirShardedServer":
        """The server from the tool's files alone: the SimplePIRConfig (a SimplePirConfig or its path) and every
        shard's prefix-i.bin and prefix-i.hint.bin, with the tool's Scalar (UInt32 for ct <= 32, else UInt64)."""
        config = config if isinstance(config, SimplePirConfig) else SimplePirConfig.load(config)
        server = SimplePirShardedServer.load(prefix, config.params, config.scalar)
        server.databaseMap = config.databaseMap
        return server

    def computeResponsesProto(self, messages) -> list:
        """One SimplePIRResponse (bytes) per SimplePIRRequest (bytes), each answered by the shard its shard_index
        names, in one device call."""
        return _responses_proto(self._h, self.shardCount, messages)

    @staticmethod
    def load(prefix: str, params: Sequence[SimplePirParameters], scalar=np.uint64) -> "SimplePirShardedServer":
        databases = [SimplePirDatabase.load(f"{prefix}-{i}.bin", p, scalar) for i, p in enumerate(params)]
        hints = [load_array2d(f"{prefix}-{i}.hint.bin", scalar) for i in range(len(params))]
        return SimplePirShardedServer(databases, hints, params, scalar)

    def close(self):
        for db in self.databases:
            db.close()


# ---- the client (SimplePir+Client.swift, SimplePir+Precompute.swift:191-356, SimplePir+Shards.swift:47-173)
def _seeds(seeds, count: int) -> np.ndarray:
    """count x 32 seed bytes; None draws them with secrets.token_bytes."""
    raw = b"".join(secrets.token_bytes(SEED_BYTES) for _ in range(count)) if seeds is None else b"".join(bytes(s) for s in seeds)
    if len(raw) != count * SEED_BYTES:
        raise PirError(f"need {count} seeds of {SEED_BYTES} bytes")
    return np.frombuffer(raw, dtype=np.uint8).copy()


@dataclass
class WithPreparedResponse:
    """PrecomputedQueries.WithPreparedResponse: the query's results (chunksPerEntry x columnSize) and index; the
    extractEntries gather runs on the device with the decryption."""
    resultsWithoutResponse: np.ndarray
    index: int


@dataclass
class WithQueryIndices:
    """PrecomputedQueries.WithQueryIndices: the request (chunksPerEntry x databaseColumns) for `index`."""
    queries: np.ndarray
    resultsWithoutResponse: np.ndarray
    index: int

    def prepareResponse(self) -> WithPreparedResponse:
        return WithPreparedResponse(self.resultsWithoutResponse, self.index)


@dataclass
class WithoutIndices:
    """PrecomputedQueries.WithoutIndices: an encrypted zero query and its resultsWithoutResponse."""
    queriesWithoutIndices: np.ndarray
    resultsWithoutResponse: np.ndarray
    params: SimplePirParameters

    def add(self, index: int) -> WithQueryIndices:
        """add(index:) (SimplePir+Precompute.swift:241-256): delta at one column per chunk, in numpy."""
        p = self.params
        ct, pt = p.ciphertextModulusBits, p.plaintextModulusBits
        q = self.queriesWithoutIndices.copy()
        dtype = q.dtype.type
        for i in range(p.chunksPerEntry):
            col = (index * p.chunksPerEntry + i) // p.entriesPerColumn
            q[i, col] = dtype((int(q[i, col]) + (1 << (ct - pt))) & ((1 << ct) - 1))
        return WithQueryIndices(q, self.resultsWithoutResponse, index)


class PrecomputedQueries:
    WithoutIndices = WithoutIndices
    WithQueryIndices = WithQueryIndices
    WithPreparedResponse = WithPreparedResponse


class DefaultQueryGenerator:
    """DefaultQueryGenerator (SimplePir+Precompute.swift:321-356) on the device: the a-polynomials (Eval) and the hint
    stay resident; addPrecomputedQueries(count) is one device call."""

    def __init__(self, params: SimplePirParameters, hint, scalar=np.uint64, errorStdDev: Optional[float] = None):
        self.scalar = np.dtype(scalar)
        bits = _word_bits(self.scalar)
        self.params = params
        hint = np.ascontiguousarray(np.asarray(hint, dtype=self.scalar))
        if hint.shape != (params.columnSize, params.latticeDimension):
            raise PirError(f"hint must be {params.columnSize} x {params.latticeDimension}, got {hint.shape}")
        if len(params.seed) != SEED_BYTES:
            raise PirError(f"seed must be {SEED_BYTES} bytes")
        cp = params._c(bits)
        cp.error_std_dev = params.encryptionParams.errorStdDev if errorStdDev is None else errorStdDev
        seed = np.frombuffer(params.seed, dtype=np.uint8).copy()
        self._h = C.c_void_p()
        _check(load_library().hecuda_simple_pir_client_create(_ptr(hint), C.byref(cp), _ptr(seed), C.byref(self._h)))
        self.unusedRequests = deque()
        self.addPrecomputedQueries()

    def precompute(self, count: int, indices=None, secretSeeds=None, errorSeeds=None):
        """count queries in one call -> (queries count x chunksPerEntry x K, results count x chunksPerEntry x M);
        with indices, WithQueryIndices.queries."""
        p = self.params
        q = np.empty((count, p.chunksPerEntry, p.databaseColumns), dtype=self.scalar)
        r = np.empty((count, p.chunksPerEntry, p.columnSize), dtype=self.scalar)
        ss, es = _seeds(secretSeeds, count), _seeds(errorSeeds, count)
        idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int64)
        if idx is not None and idx.shape != (count,):
            raise PirError("one index per query")
        _check(load_library().hecuda_simple_pir_client_precompute(self._h, _ptr(ss), _ptr(es),
                                                                  None if idx is None else _ptr(idx), count, _ptr(q), _ptr(r)))
        return q, r

    def addPrecomputedQueries(self, count: int = 1):
        q, r = self.precompute(count)
        self.unusedRequests.extend(WithoutIndices(q[i], r[i], self.params) for i in range(count))

    def nextPrecomputedQueries(self) -> WithoutIndices:
        if self.unusedRequests:
            return self.unusedRequests.popleft()
        q, r = self.precompute(1)
        return WithoutIndices(q[0], r[0], self.params)

    def close(self):
        if self._h is not None:
            load_library().hecuda_simple_pir_client_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SimplePirClient:
    """SimplePirClient<DefaultQueryGenerator> (SimplePir+Client.swift:98-127) with batched forms."""

    def __init__(self, queryGenerator: DefaultQueryGenerator):
        self.queryGenerator = queryGenerator
        self.params, self.scalar = queryGenerator.params, queryGenerator.scalar

    def query(self, at: int) -> WithQueryIndices:
        return self.queryGenerator.nextPrecomputedQueries().add(at)

    def queries(self, indices, secretSeeds=None, errorSeeds=None):
        """One precompute call with the deltas added on the device -> [WithQueryIndices]."""
        indices = [int(i) for i in indices]
        q, r = self.queryGenerator.precompute(len(indices), indices, secretSeeds, errorSeeds)
        return [WithQueryIndices(q[i], r[i], ix) for i, ix in enumerate(indices)]

    def decryptMany(self, responses, results, indices) -> np.ndarray:
        """count responses (count x chunksPerEntry x columnSize) -> count x entrySizeInBytes bytes, one device call."""
        p = self.params
        resp = np.ascontiguousarray(np.asarray(responses, dtype=self.scalar)).reshape(-1, p.chunksPerEntry, p.columnSize)
        res = np.ascontiguousarray(np.asarray(results, dtype=self.scalar)).reshape(resp.shape)
        idx = np.ascontiguousarray(indices, dtype=np.int64).reshape(-1)
        if idx.shape[0] != resp.shape[0]:
            raise PirError("one index per response")
        out = np.empty((resp.shape[0], p.entrySizeInBytes), dtype=np.uint8)
        _check(load_library().hecuda_simple_pir_client_decrypt(self.queryGenerator._h, _ptr(resp), _ptr(res), _ptr(idx),
                                                               resp.shape[0], _ptr(out)))
        return out

    def decrypt(self, responses, with_: WithPreparedResponse, at: int) -> bytes:
        return self.decryptMany(responses[None], with_.resultsWithoutResponse[None], [at])[0].tobytes()

    def precomputeDevice(self, secret_seeds_ptr: int, error_seeds_ptr: int, indices_ptr: Optional[int], count: int,
                         queries_ptr: int, results_ptr: int, stream: int = 0):
        """Device buffers (torch data_ptr()): enqueue on `stream` without synchronising."""
        _check(load_library().hecuda_simple_pir_client_precompute_device(
            self.queryGenerator._h, C.c_void_p(secret_seeds_ptr), C.c_void_p(error_seeds_ptr),
            None if indices_ptr is None else C.c_void_p(indices_ptr), count, C.c_void_p(queries_ptr),
            C.c_void_p(results_ptr), C.c_void_p(stream)))

    def decryptDevice(self, responses_ptr: int, results_ptr: int, indices_ptr: int, count: int, entries_ptr: int,
                      stream: int = 0):
        _check(load_library().hecuda_simple_pir_client_decrypt_device(
            self.queryGenerator._h, C.c_void_p(responses_ptr), C.c_void_p(results_ptr), C.c_void_p(indices_ptr), count,
            C.c_void_p(entries_ptr), C.c_void_p(stream)))


class SimplePirClientForAllShards:
    """SimplePirClientForAllShards (SimplePir+Shards.swift:47-173): one SimplePirClient per shard."""

    def __init__(self, databaseMap, clients: Sequence[SimplePirClient]):
        self.shardMap = databaseMap if isinstance(databaseMap, ShardMap) else ShardMap(databaseMap)
        self.clients = list(clients)
        if self.shardMap.shardCount != len(self.clients):
            raise PirError(f"validationError: Mismatching shard count {self.shardMap.shardCount} and number of clients "
                           f"{len(self.clients)}")

    @property
    def queriesPerShard(self) -> int:
        return self.shardMap.chunksPerShard

    def _rows(self, index: int):
        rows = [[] for _ in self.clients]
        entry = self.shardMap[index]
        if entry is not None:
            for c in entry.chunks:
                rows[c.shardIndex].append(c.index)
        return [r + [0] * (self.shardMap.chunksPerShard - len(r)) for r in rows]

    def query(self, index: int):
        """query(for:): per shard chunksPerShard WithQueryIndices (the entry's rows, then row 0), one precompute call
        per shard; an absent index makes the same calls with the same shapes."""
        return [client.queries(rows) for client, rows in zip(self.clients, self._rows(index))]

    def queriesMany(self, indices):
        """query(for:) for many clients at once -> (count x words requests in the client-major layout
        SimplePirShardedServer.computeResponses(..., requests_per_shard) reads, the per-shard [WithQueryIndices] lists)."""
        per = self.shardMap.chunksPerShard
        rows = [self._rows(int(i)) for i in indices]
        shards = [self.clients[s].queries([r for client in rows for r in client[s]]) for s in range(len(self.clients))]
        flat = np.stack([np.concatenate([np.stack([w.queries for w in shards[s][c * per:(c + 1) * per]]).reshape(-1)
                                         for s in range(len(self.clients))]) for c in range(len(rows))])
        return flat, [[shards[s][c * per:(c + 1) * per] for s in range(len(self.clients))] for c in range(len(rows))]

    def decrypt(self, responses, index: int, queries) -> Optional[bytes]:
        """decrypt(responses:for:with:): every query of every shard is decrypted (one device call per shard), then the
        reference's fixed-work chunk selection; None for an index the map does not hold."""
        if len(responses) != len(self.clients) or len(queries) != len(self.clients):
            raise PirError("validationError: one response and query list per shard")
        plain = []
        for client, rs, qs in zip(self.clients, responses, queries):
            if len(rs) != len(qs):
                raise PirError("validationError: response count does not match query count")
            plain.append(client.decryptMany(np.stack([np.asarray(r) for r in rs]),
                                            np.stack([q.resultsWithoutResponse for q in qs]), [q.index for q in qs]))
        entry = self.shardMap[index]
        chunks = entry.chunks if entry is not None else ()
        out = b""
        for c in range(self.shardMap.maximumChunkCount):
            real = c < len(chunks)
            shard, row = (chunks[c].shardIndex, chunks[c].index) if real else (0, 0)
            at = 0
            for i, q in enumerate(queries[shard]):
                at = i if q.index == row else at
            out += plain[shard][at][:self.shardMap.chunkSize].tobytes()
        return None if entry is None else out[:entry.size]


def _sharded_client_from_config(prefix: str, config, errorStdDev: Optional[float] = None) -> "SimplePirClientForAllShards":
    """SimplePirClientForAllShards from the tool's files alone: the config (or its path) and every prefix-i.hint.bin."""
    config = config if isinstance(config, SimplePirConfig) else SimplePirConfig.load(config)
    clients = [SimplePirClient(DefaultQueryGenerator(p, load_array2d(f"{prefix}-{i}.hint.bin", config.scalar), config.scalar,
                                                     errorStdDev)) for i, p in enumerate(config.params)]
    return SimplePirClientForAllShards(config.databaseMap, clients)


def _request_messages(self, index: int, configurationHash: bytes = b""):
    """query(for:) as SimplePIRRequests: one message per shard s holding its chunksPerShard x chunksPerEntry_s rows of
    K_s words, stacked -> (messages, the per-shard [WithQueryIndices] lists for decryptResponseMessages)."""
    queries = self.query(index)
    messages = []
    for s, (client, qs) in enumerate(zip(self.clients, queries)):
        words = np.concatenate([q.queries.reshape(-1, client.params.databaseColumns) for q in qs])
        messages.append(SimplePirRequest.write(words, s, configurationHash))
    return messages, queries


def _decrypt_response_messages(self, messages, index: int, queries) -> Optional[bytes]:
    """decrypt(responses:for:with:) from one SimplePIRResponse per shard (each chunksPerShard x chunksPerEntry_s rows of
    M_s words); None for an index the map does not hold."""
    if len(messages) != len(self.clients):
        raise PirError("validationError: one response message per shard")
    responses = []
    for client, message, qs in zip(self.clients, messages, queries):
        p = client.params
        words = SimplePirResponse.read(message, client.scalar)
        if words.shape != (len(qs) * p.chunksPerEntry, p.columnSize):
            raise PirError(f"validationError: a response of {words.shape}, expected "
                           f"{(len(qs) * p.chunksPerEntry, p.columnSize)}")
        responses.append(list(words.reshape(len(qs), p.chunksPerEntry, p.columnSize)))
    return self.decrypt(responses, index, queries)


SimplePirClientForAllShards.fromConfig = staticmethod(_sharded_client_from_config)
SimplePirClientForAllShards.requestMessages = _request_messages
SimplePirClientForAllShards.decryptResponseMessages = _decrypt_response_messages


# ---- protobuf messages (api/pir/v1/pir.proto, pir/v1/simple_pir.proto; PirConversion.swift:380-518)
class _RequestFields(C.Structure):  # hecuda_simple_pir_request_fields
    _fields_ = [("has_request", C.c_int32), ("row_count", C.c_uint32), ("col_count", C.c_uint32),
                ("shard_index", C.c_uint32), ("data_run_count", C.c_int64), ("data_bytes", C.c_uint64),
                ("configuration_hash_offset", C.c_uint64), ("configuration_hash_bytes", C.c_uint64)]


class _ConfigShape(C.Structure):  # hecuda_simple_pir_config_shape
    _fields_ = [("entry_count", C.c_int64), ("chunk_count", C.c_int64), ("chunk_size", C.c_uint64),
                ("shard_count", C.c_int32), ("hint_identifier_count", C.c_int32)]


def _bytes_arg(data: bytes):
    data = bytes(data)
    return C.create_string_buffer(data, max(len(data), 1)), len(data)


def _responses_proto(handles, shard_count: int, messages) -> list:
    messages = [bytes(m) for m in messages]
    if not messages:
        return []
    # the messages are read in place (c_char_p points into each bytes object, which `messages` keeps alive)
    ptrs = (C.c_void_p * len(messages))(*[C.cast(C.c_char_p(m), C.c_void_p).value for m in messages])
    sizes = np.array([len(m) for m in messages], dtype=np.uint64)
    lib = load_library()
    caps = np.zeros(len(messages), dtype=np.uint64)
    _check(lib.hecuda_simple_pir_response_proto_byte_count(handles, shard_count, ptrs, _ptr(sizes), len(messages),
                                                           _ptr(caps)))
    offsets = np.zeros(len(messages), dtype=np.uint64)
    offsets[1:] = np.cumsum(caps)[:-1]
    out = np.empty(max(int(caps.sum()), 1), dtype=np.uint8)
    lengths = np.zeros(len(messages), dtype=np.uint64)
    _check(lib.hecuda_simple_pir_compute_response_proto(handles, shard_count, ptrs, _ptr(sizes), len(messages), _ptr(out),
                                                        _ptr(offsets), _ptr(lengths)))
    return [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(offsets, lengths)]


class SimplePirRequest:
    """api.pir.v1.SimplePIRRequest."""

    @staticmethod
    def fields(message: bytes) -> dict:
        """The walk of one request (data located, not read): has_request, row_count, col_count, shard_index,
        data_run_count, data_bytes and configuration_hash."""
        buf, n = _bytes_arg(message)
        f = _RequestFields()
        _check(load_library().hecuda_simple_pir_request_fields_read(buf, n, C.byref(f)))
        at, size = f.configuration_hash_offset, f.configuration_hash_bytes
        return {"has_request": bool(f.has_request), "row_count": f.row_count, "col_count": f.col_count,
                "shard_index": f.shard_index, "data_run_count": f.data_run_count, "data_bytes": f.data_bytes,
                "configuration_hash": bytes(message)[at:at + size]}

    @staticmethod
    def write(words, shardIndex: int = 0, configurationHash: bytes = b"") -> bytes:
        """Array2d.proto() of a rows x columns word matrix in a SimplePIRRequest, data packed."""
        w = np.ascontiguousarray(np.asarray(words), dtype=np.uint64)
        if w.ndim != 2:
            raise PirError("a request is a rows x columns word matrix")
        h, hn = _bytes_arg(configurationHash)
        lib, written = load_library(), C.c_uint64(0)
        data = w if w.size else np.zeros(1, dtype=np.uint64)
        _check(lib.hecuda_simple_pir_request_write(w.shape[0], w.shape[1], _ptr(data), shardIndex, h, hn, None, 0,
                                                   C.byref(written)))
        out = np.empty(max(written.value, 1), dtype=np.uint8)
        _check(lib.hecuda_simple_pir_request_write(w.shape[0], w.shape[1], _ptr(data), shardIndex, h, hn, _ptr(out),
                                                   written.value, C.byref(written)))
        return out[:written.value].tobytes()


class SimplePirResponse:
    """api.pir.v1.SimplePIRResponse."""

    @staticmethod
    def read(message: bytes, scalar=np.uint64) -> np.ndarray:
        """SimplePIRMatrix.native(): the rows x columns words (a value the scalar cannot hold is refused, where the
        reference's Scalar(_:) traps)."""
        buf, n = _bytes_arg(message)
        rows, cols = C.c_uint32(0), C.c_uint32(0)
        lib = load_library()
        # every value takes one byte at least, so the message's size bounds the count
        data = np.empty(max(n, 1), dtype=np.uint64)
        _check(lib.hecuda_simple_pir_response_read(buf, n, C.byref(rows), C.byref(cols), _ptr(data), n))
        words = data[:rows.value * cols.value]
        if np.dtype(scalar) == np.dtype(np.uint32) and words.size and int(words.max()) >> 32:
            raise PirError("SimplePIRMatrix: a value at or above 2^32 for UInt32")
        return words.astype(scalar).reshape(rows.value, cols.value)


class SimplePirConfig:
    """api.pir.v1.SimplePIRConfig: the databaseMap, one SimplePirParameters per shard and one hint identifier (SHA-256
    of the hint file) per shard, as the SimplePIRProcessDatabase tool writes them (main.swift:231-240)."""

    def __init__(self, databaseMap: DatabaseMap, params: Sequence[SimplePirParameters], hintIdentifiers: Sequence[bytes]):
        self.databaseMap, self.params = databaseMap, list(params)
        self.hintIdentifiers = [bytes(h) for h in hintIdentifiers]

    @property
    def scalar(self):
        """The tool's Scalar: UInt32 for ct <= 32, else UInt64 (main.swift:369-371)."""
        return np.uint32 if self.params and self.params[0].ciphertextModulusBits <= 32 else np.uint64

    def __eq__(self, other):
        return (isinstance(other, SimplePirConfig) and self.databaseMap == other.databaseMap and
                self.params == other.params and self.hintIdentifiers == other.hintIdentifiers)

    def _args(self):
        m = self.databaseMap
        counts = ((m.sizes + m.chunkSize - 1) // m.chunkSize).astype(np.uint64)
        index = np.ascontiguousarray(m.originalIndices.astype(np.uint64))
        sizes = np.ascontiguousarray(m.sizes.astype(np.uint64))
        locs = np.ascontiguousarray(m.chunkLocations, dtype=np.int64)
        cparams = (_Params * max(len(self.params), 1))(*[p._c(32 if p.ciphertextModulusBits <= 32 else 64)
                                                          for p in self.params])
        seeds = np.frombuffer(b"".join(p.seed for p in self.params) or b"\0", dtype=np.uint8).copy()
        ids = [C.create_string_buffer(h, max(len(h), 1)) for h in self.hintIdentifiers]
        id_ptrs = (C.c_void_p * max(len(ids), 1))(*[C.addressof(b) for b in ids])
        id_sizes = np.array([len(h) for h in self.hintIdentifiers] or [0], dtype=np.uint64)
        keep = (index, sizes, counts, locs, cparams, seeds, ids, id_ptrs, id_sizes)
        args = [_ptr(index), _ptr(sizes), _ptr(counts), len(sizes), _ptr(locs), m.chunkSize, cparams, _ptr(seeds),
                len(self.params), id_ptrs, _ptr(id_sizes), len(self.hintIdentifiers)]
        return keep, args

    def serialize(self) -> bytes:
        for p in self.params:
            if len(p.seed) != SEED_BYTES:
                raise PirError(f"seed must be {SEED_BYTES} bytes")
        keep, args = self._args()
        lib, n = load_library(), C.c_uint64(0)
        _check(lib.hecuda_simple_pir_config_serialized_byte_count(*args, C.byref(n)))
        out = np.empty(max(n.value, 1), dtype=np.uint8)
        _check(lib.hecuda_simple_pir_config_serialize(*args, _ptr(out), n.value))
        del keep
        return out[:n.value].tobytes()

    @staticmethod
    def deserialize(data: bytes, securityLevel: str = "quantum128") -> "SimplePirConfig":
        """SimplePIRConfig -> its fields, refused as the reference's native() refuses (errorStdDev, a_seed) and as the
        library refuses parameters; each shard's encryption parameters are checked at securityLevel."""
        buf, n = _bytes_arg(data)
        lib, shape = load_library(), _ConfigShape()
        _check(lib.hecuda_simple_pir_config_describe(buf, n, C.byref(shape)))
        entries, chunks, shards = shape.entry_count, shape.chunk_count, shape.shard_count
        index, sizes, counts = (np.zeros(max(entries, 1), dtype=np.uint64) for _ in range(3))
        locs = np.zeros((max(chunks, 1), 2), dtype=np.int64)
        cparams = (_Params * max(shards, 1))()
        seeds = np.zeros(max(shards, 1) * SEED_BYTES, dtype=np.uint8)
        ranges = np.zeros((max(shape.hint_identifier_count, 1), 2), dtype=np.uint64)
        _check(lib.hecuda_simple_pir_config_read(buf, n, _ptr(index), _ptr(sizes), _ptr(counts), _ptr(locs), cparams,
                                                 _ptr(seeds), _ptr(ranges)))
        size = sizes[:entries].astype(np.int64)
        chunk_size = int(shape.chunk_size)
        if chunk_size < 1 and chunks:
            raise PirError("DatabaseMapping: chunk_size must be positive")
        if entries and not np.array_equal(counts[:entries].astype(np.int64), (size + max(chunk_size, 1) - 1) // max(chunk_size, 1)):
            raise PirError("DatabaseMapping: an entry's chunk count is not ceil(size / chunk_size)")
        database_map = DatabaseMap(index[:entries].astype(np.int64), size, locs[:chunks], chunk_size)
        params = []
        for s in range(shards):
            c = cparams[s]
            enc = SimplePirEncryptionParams(c.plaintext_modulus_bits, c.ciphertext_modulus_bits, c.lattice_dimension,
                                            c.error_std_dev, securityLevel)
            params.append(SimplePirParameters(enc, c.entry_size, c.entries_per_column, c.chunks_per_entry,
                                              c.database_columns, seeds[SEED_BYTES * s:SEED_BYTES * (s + 1)].tobytes()))
        raw = bytes(data)
        ids = [raw[int(a):int(a) + int(b)] for a, b in ranges[:shape.hint_identifier_count]]
        return SimplePirConfig(database_map, params, ids)

    def save(self, path: str):
        with open(path, "wb") as f:
            f.write(self.serialize())

    @staticmethod
    def load(path: str, securityLevel: str = "quantum128") -> "SimplePirConfig":
        with open(path, "rb") as f:
            return SimplePirConfig.deserialize(f.read(), securityLevel)


def _validate(trial, trials: int, index: int, expected: bytes):
    """verifyProcessing (SimplePIRProcessDatabase/main.swift:260-348): `trials` fresh queries for `index`."""
    times, value = [], None
    for _ in range(trials):
        start = time.perf_counter()
        value = trial()
        times.append(time.perf_counter() - start)
        if value != bytes(expected):
            raise PirError(f"Verification failed for index {index}")
    return times, value


def _server_validate(self, row, trials: int = 1, errorStdDev: Optional[float] = None):
    """Query, answer and decrypt entry `row` = (index, expected bytes) with a device client built from the hint; raise
    PirError on a mismatch.  -> (seconds per round trip, decrypted bytes)."""
    index, expected = row
    client = SimplePirClient(DefaultQueryGenerator(self.params, self.hint, self.scalar, errorStdDev))

    def trial():
        q = client.queries([index])[0]
        response = self.computeResponse(q.queries)
        return client.decrypt(response, q.prepareResponse(), index)

    try:
        return _validate(trial, trials, index, expected)
    finally:
        client.queryGenerator.close()


def _sharded_validate(self, row, databaseMap: Optional[DatabaseMap] = None, trials: int = 1,
                      errorStdDev: Optional[float] = None):
    """verifyProcessing for sharded databases: entry `row` = (originalIndex, expected bytes) through one device client
    per shard built from its hint and the all-shards client; raise PirError on a mismatch.  -> (seconds per round
    trip, decrypted bytes)."""
    index, expected = row
    database_map = databaseMap if databaseMap is not None else self.databaseMap
    if database_map is None:
        raise PirError("validate needs the databaseMap")
    clients = [SimplePirClient(DefaultQueryGenerator(p, h, self.scalar, errorStdDev)) for p, h in zip(self.params, self.hints)]
    all_shards = SimplePirClientForAllShards(database_map, clients)
    per = all_shards.queriesPerShard

    def trial():
        flat, queries = all_shards.queriesMany([index])
        out = self.computeResponses(flat, requests_per_shard=per)[0]
        bounds = np.concatenate([[0], np.cumsum(self._words(per)[1])])
        responses = [out[bounds[s]:bounds[s + 1]].reshape(per, p.chunksPerEntry, p.columnSize)
                     for s, p in enumerate(self.params)]
        return all_shards.decrypt(responses, index, queries[0])

    try:
        return _validate(trial, trials, index, expected)
    finally:
        for c in clients:
            c.queryGenerator.close()


SimplePirServer.validate = _server_validate
SimplePirShardedServer.validate = _sharded_validate
