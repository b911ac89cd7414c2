"""hecuda.keyword_pir -- the reference's keyword PIR server over libhecuda.

Names and argument meaning follow Sources/PrivateInformationRetrieval/KeywordPir:

    CuckooTableConfig, CuckooTable                 CuckooTable.swift
    HashKeyword.hash / hashIndices                 HashBucket.swift:208-270
    KeywordDatabase, ShardingFunction, Sharding    KeywordDatabase.swift
    KeywordPirConfig, KeywordPirParameter          KeywordPirProtocol.swift:19-114
    KeywordPirServer.process / computeResponse     KeywordPirProtocol.swift:137-276
    KeywordPirClient                               KeywordPirProtocol.swift:280-392
    KeywordDatabase.validateShard                  KeywordDatabase.swift:557-630
    KeywordDatabase.symmetricPIRProcess            SymmetricPir/SymmetricPirDatabase.swift:186-211 (hecuda.symmetric_pir)

Keyword hashing, candidate indices and bucket serialization run on the device; the cuckoo placement runs on the host
inside libhecuda (csrc/cuckoo.hpp) because the table depends on the order of its random draws.  The table's buckets
are serialized, packed and converted to Eval on the device, one MulPir database per hash function, and answered by
MulPirServer with indicesCount = hashFunctionCount.

One deliberate divergence from the reference (csrc/cuckoo.hpp, include/hecuda.h): when no candidate bucket has a swap
index, CuckooTable.insertLoop expands and drops the pair in hand; here that pair is inserted again after the expansion.
"""
from __future__ import annotations

import ctypes as C
import struct
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import Context, EvaluationKey, SecretKey, _check, _ptr, load_library
from . import symmetric_pir
from .pir import IndexPirConfig, IndexPirParameter, MulPir, MulPirClient, MulPirServer, PirError, PirKeyCompressionStrategy, \
    PirWire, ProcessedDatabase, ShardValidationResult, _save_databases, _validate, bytesPerPlaintext, responseFromMessage
from .symmetric_pir import SymmetricPirClientConfig, SymmetricPirConfig

MAX_SLOT_COUNT = 255  # HashBucket.maxSlotCount
RNG_COUNTER, RNG_SPLITMIX64 = 0, 1  # HECUDA_CUCKOO_RNG_*

KeywordValuePair = Tuple[bytes, bytes]


class _Config(C.Structure):
    _fields_ = [("hash_function_count", C.c_int32), ("max_eviction_count", C.c_int64),
                ("max_serialized_bucket_size", C.c_int64), ("slot_count", C.c_int32), ("multiple_tables", C.c_int32),
                ("fixed_bucket_count", C.c_int64), ("expansion_factor", C.c_double), ("target_load_factor", C.c_double)]


class _Summary(C.Structure):
    _fields_ = [("entry_count", C.c_int64), ("bucket_count", C.c_int64), ("buckets_per_table", C.c_int64),
                ("empty_bucket_count", C.c_int64), ("serialized_bytes", C.c_int64),
                ("max_serialized_bucket_size", C.c_int64)]


def _concatenate(blobs: Sequence[bytes]):
    """Rows as the C ABI takes them: concatenated bytes and count + 1 offsets."""
    blobs = [bytes(b) for b in blobs]
    offsets = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    data = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)
    return data, offsets


def serializedSize(singleValueSize: int) -> int:
    """HashBucket.serializedSize(singleValueSize:): slot count + keyword hash + value length + value."""
    return 1 + 8 + 2 + singleValueSize


# ------------------------------------------------------------------------------------------------ hashing
class HashKeyword:
    """enum HashKeyword (HashBucket.swift:208-270), on the device for many keywords at once."""

    @staticmethod
    def hashes(keywords: Sequence[bytes]) -> np.ndarray:
        """HashKeyword.hash of every keyword (first 8 bytes of SHA-256, little-endian) -> (count,) uint64."""
        data, offsets = _concatenate(keywords)
        out = np.empty(len(offsets) - 1, dtype=np.uint64)
        _check(load_library().hecuda_keyword_hash(_ptr(data), _ptr(offsets), len(out), _ptr(out)))
        return out

    @staticmethod
    def hashIndicesOfHashes(hashes, bucketCount: int, hashFunctionCount: int) -> np.ndarray:
        h = np.ascontiguousarray(np.asarray(hashes, dtype=np.uint64).reshape(-1))
        out = np.empty((h.size, hashFunctionCount), dtype=np.int64)
        _check(load_library().hecuda_keyword_hash_indices(_ptr(h), h.size, bucketCount, hashFunctionCount, _ptr(out)))
        return out

    @staticmethod
    def hashIndices(keyword: bytes, bucketCount: int, hashFunctionCount: int) -> List[int]:
        """HashKeyword.hashIndices (HashBucket.swift:221-235) of one keyword."""
        return [int(i) for i in HashKeyword.hashIndicesOfHashes(HashKeyword.hashes([keyword]), bucketCount,
                                                                 hashFunctionCount)[0]]


class HashBucket:
    """HashBucket (HashBucket.swift): a serialized bucket is a slot count, then per slot the keyword hash (UInt64), the
    value length (UInt16), both little-endian, and the value."""

    @staticmethod
    def deserialize(raw: bytes) -> List[Tuple[int, bytes]]:
        """HashBucket(deserialize:) -> [(keyword hash, value)]; PirError("corruptedData...") on a short buffer."""
        if not raw:
            raise PirError("corruptedData: Serialized HashBucket shouldn't be empty.")
        count, offset, slots = raw[0], 1, []
        for _ in range(count):
            if len(raw) < offset + 10:
                raise PirError("corruptedData: Serialized HashBucketEntry should at least have a keyword hash and a value size.")
            keyword_hash, size = struct.unpack_from("<QH", raw, offset)
            offset += 10
            if offset + size > len(raw):
                raise PirError("corruptedData: HashBucketEntry buffer has less data than expected")
            slots.append((keyword_hash, bytes(raw[offset:offset + size])))
            offset += size
        return slots

    @staticmethod
    def serializedSize(slots: Sequence[Tuple[int, bytes]]) -> int:
        return 1 + sum(10 + len(value) for _, value in slots)

    @staticmethod
    def find(slots: Sequence[Tuple[int, bytes]], keywordHash: int) -> Optional[bytes]:
        for slot_hash, value in slots:
            if slot_hash == keywordHash:
                return value
        return None


# ------------------------------------------------------------------------------------------------ cuckoo table
@dataclass(frozen=True)
class AllowExpansion:
    """CuckooTableConfig.BucketCountConfig.allowExpansion."""

    expansionFactor: float
    targetLoadFactor: float


@dataclass(frozen=True)
class FixedSize:
    """CuckooTableConfig.BucketCountConfig.fixedSize."""

    bucketCount: int


@dataclass(frozen=True)
class CuckooTableConfig:
    """CuckooTableConfig (CuckooTable.swift:19-157)."""

    hashFunctionCount: int
    maxEvictionCount: int
    maxSerializedBucketSize: int
    bucketCount: Union[AllowExpansion, FixedSize]
    multipleTables: bool = True
    slotCount: int = MAX_SLOT_COUNT

    def __post_init__(self):  # validate (:138-156)
        ok = (self.hashFunctionCount > 0 and self.maxSerializedBucketSize >= serializedSize(0)
              and 0 < self.slotCount <= MAX_SLOT_COUNT)
        if isinstance(self.bucketCount, AllowExpansion):
            ok = ok and self.bucketCount.expansionFactor > 1.0 and self.bucketCount.targetLoadFactor < 1.0
        else:
            ok = ok and self.maxSerializedBucketSize > 0 and self.bucketCount.bucketCount > 0
        if not ok:
            raise PirError(f"invalidCuckooConfig(config: {self})")

    @staticmethod
    def defaultKeywordPir(maxSerializedBucketSize: int) -> "CuckooTableConfig":
        return CuckooTableConfig(2, 100, maxSerializedBucketSize, AllowExpansion(1.1, 0.9))

    def freezingTableSize(self, maxSerializedBucketSize: int, bucketCount: int) -> "CuckooTableConfig":
        """A fixed-size copy; like the reference (:127-134) it keeps the default slot count."""
        return CuckooTableConfig(self.hashFunctionCount, self.maxEvictionCount, maxSerializedBucketSize,
                                 FixedSize(bucketCount), self.multipleTables)

    @property
    def tableCount(self) -> int:
        return self.hashFunctionCount if self.multipleTables else 1

    def _c(self) -> _Config:
        expand = isinstance(self.bucketCount, AllowExpansion)
        return _Config(self.hashFunctionCount, self.maxEvictionCount, self.maxSerializedBucketSize, self.slotCount,
                       1 if self.multipleTables else 0, 0 if expand else self.bucketCount.bucketCount,
                       self.bucketCount.expansionFactor if expand else 0.0,
                       self.bucketCount.targetLoadFactor if expand else 0.0)


@dataclass(frozen=True)
class CuckooTableInformation:
    """CuckooTable.CuckooTableInformation (:259-270)."""

    entryCount: int
    bucketCount: int
    emptyBucketCount: int
    loadFactor: np.float32


@dataclass(frozen=True)
class Rng:
    """The generator of the table's evictions: `counter(seed)` is the reference's TestRng(counter: seed);
    `splitMix64(seed)` is the one to use in production."""

    kind: int
    seed: int

    @staticmethod
    def counter(seed: int = 0) -> "Rng":
        return Rng(RNG_COUNTER, seed)

    @staticmethod
    def splitMix64(seed: int = 0) -> "Rng":
        return Rng(RNG_SPLITMIX64, seed)


class CuckooTable:
    """CuckooTable(config:database:using:) (CuckooTable.swift:328-357) built by libhecuda; the values stay on the
    device with it."""

    def __init__(self, context: Context, config: CuckooTableConfig, database: Sequence[KeywordValuePair],
                 rng: Rng = Rng.splitMix64()):
        self.context, self.config = context, config
        keywords, koff = _concatenate([k for k, _ in database])
        values, voff = _concatenate([v for _, v in database])
        cfg = config._c()
        h = C.c_void_p()
        _check(load_library().hecuda_cuckoo_table_create(context._h, _ptr(keywords), _ptr(koff), _ptr(values), _ptr(voff),
                                                         len(koff) - 1, C.byref(cfg), rng.kind, rng.seed & ((1 << 64) - 1),
                                                         C.byref(h)))
        self._h = h
        s = _Summary()
        _check(load_library().hecuda_cuckoo_table_summarize(self._h, C.byref(s)))
        self._summary = s

    @property
    def bucketCount(self) -> int:
        return self._summary.bucket_count

    @property
    def bucketsPerTable(self) -> int:
        return self._summary.buckets_per_table

    @property
    def entryCount(self) -> int:
        return self._summary.entry_count

    def summarize(self) -> CuckooTableInformation:
        s = self._summary
        load = np.float32(s.serialized_bytes) / np.float32(s.bucket_count * self.config.maxSerializedBucketSize)
        return CuckooTableInformation(s.entry_count, s.bucket_count, s.empty_bucket_count, load)

    def maxSerializedBucketSize(self) -> int:
        return self._summary.max_serialized_bucket_size

    def serializedBucketBytes(self):
        """(bytes, bucketCount + 1 offsets) of serializeBuckets(), written on the device."""
        data = np.empty(max(self._summary.serialized_bytes, 1), dtype=np.uint8)
        offsets = np.empty(self._summary.bucket_count + 1, dtype=np.uint64)
        _check(load_library().hecuda_cuckoo_table_serialize_buckets(self._h, _ptr(data), data.size, _ptr(offsets)))
        return data, offsets

    def serializeBuckets(self) -> List[bytes]:
        """CuckooTable.serializeBuckets() (:376-378)."""
        data, offsets = self.serializedBucketBytes()
        raw = data.tobytes()
        return [raw[int(offsets[b]):int(offsets[b + 1])] for b in range(len(offsets) - 1)]

    def close(self):
        if getattr(self, "_h", None) is not None:
            load_library().hecuda_cuckoo_table_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------ sharding
@dataclass(frozen=True)
class ShardingFunction:
    """ShardingFunction (KeywordDatabase.swift:65-112): sha256, or doubleMod(otherShardCount)."""

    otherShardCount: Optional[int] = None

    @staticmethod
    def doubleMod(otherShardCount: int) -> "ShardingFunction":
        return ShardingFunction(otherShardCount)

    def shardIndices(self, hashes: np.ndarray, shardCount: int) -> np.ndarray:
        """shardIndex(keyword:shardCount:) from HashKeyword.hashes of the keywords."""
        h = np.asarray(hashes, dtype=np.uint64)
        if self.otherShardCount is not None:
            h = h % np.uint64(self.otherShardCount)
        return (h % np.uint64(shardCount)).astype(np.int64)


ShardingFunction.sha256 = ShardingFunction()


@dataclass(frozen=True)
class Sharding:
    """Sharding (KeywordDatabase.swift:150-268): shardCount(n) or entryCountPerShard(n)."""

    shardCountValue: Optional[int] = None
    entryCountPerShardValue: Optional[int] = None

    @staticmethod
    def shardCount(count: int) -> "Sharding":
        return Sharding(shardCountValue=count)

    @staticmethod
    def entryCountPerShard(count: int) -> "Sharding":
        return Sharding(entryCountPerShardValue=count)

    def shardCountFor(self, rowCount: int) -> int:
        if self.shardCountValue is not None:
            return self.shardCountValue
        return max(rowCount // self.entryCountPerShardValue, 1)


class KeywordDatabase:
    """KeywordDatabase (KeywordDatabase.swift:388-437): rows split into shards by their device-computed keyword hashes.
    shards: shard id (str) -> [(keyword, value)] in row order.  With a symmetricPirConfig the rows are first replaced by
    symmetricPIRProcess's (keyword', sealed value) rows, and those are sharded; the shard count still comes from the row
    count."""

    def __init__(self, rows: Sequence[KeywordValuePair], sharding: Sharding,
                 shardingFunction: ShardingFunction = ShardingFunction.sha256,
                 symmetricPirConfig: Optional[SymmetricPirConfig] = None):
        rows = [(bytes(k), bytes(v)) for k, v in rows]
        count = sharding.shardCountFor(len(rows))
        if symmetricPirConfig is not None:
            rows = KeywordDatabase.symmetricPIRProcess(rows, symmetricPirConfig)
        indices = shardingFunction.shardIndices(HashKeyword.hashes([k for k, _ in rows]), count) if rows else []
        shards: Dict[str, Dict[bytes, bytes]] = {}
        for (keyword, value), index in zip(rows, indices):
            shard = shards.setdefault(str(int(index)), {})
            if keyword in shard:  # Dictionary.updateValue returned the previous value (:421-433)
                raise PirError(f"invalidDatabaseDuplicateKeyword(keyword: {list(keyword)}, oldValue: {list(shard[keyword])}, "
                               f"newValue: {list(value)})")
            shard[keyword] = value
        self.shards = {sid: list(rows.items()) for sid, rows in shards.items()}

    @staticmethod
    def symmetricPIRProcess(database: Sequence[KeywordValuePair], config: SymmetricPirConfig) -> List[KeywordValuePair]:
        """KeywordDatabase.symmetricPIRProcess(database:config:) (SymmetricPirDatabase.swift:193-211), every row on the
        device: (keyword, value) -> (OPRF output[0:16], AES-GCM-192 ciphertext || tag)."""
        return symmetric_pir.symmetricPIRProcess(database, config)


# ------------------------------------------------------------------------------------------------ keyword PIR
@dataclass(frozen=True)
class KeywordPirParameter:
    """KeywordPirParameter (KeywordPirProtocol.swift:91-114)."""

    hashFunctionCount: int
    shardingFunction: ShardingFunction = ShardingFunction.sha256


@dataclass
class KeywordPirConfig:
    """KeywordPirConfig (KeywordPirProtocol.swift:19-86)."""

    dimensionCount: int
    cuckooTableConfig: CuckooTableConfig
    unevenDimensions: bool
    keyCompression: PirKeyCompressionStrategy
    useMaxSerializedBucketSize: bool = False
    shardingFunction: ShardingFunction = ShardingFunction.sha256
    symmetricPirClientConfig: Optional[SymmetricPirClientConfig] = None

    def __post_init__(self):
        if self.dimensionCount not in (1, 2):
            raise PirError(f"invalidDimensionCount(dimensionCount: {self.dimensionCount}, expected: [1, 2])")
        if not self.cuckooTableConfig.multipleTables:
            raise PirError(f"invalidCuckooConfig(config: {self.cuckooTableConfig})")
        self.keyCompression = PirKeyCompressionStrategy(self.keyCompression)

    @property
    def parameter(self) -> KeywordPirParameter:
        return KeywordPirParameter(self.cuckooTableConfig.hashFunctionCount, self.shardingFunction)


@dataclass
class ProcessedKeywordDatabase:
    """ProcessedDatabaseWithParameters of a keyword database: one resident MulPir database per hash function."""

    databases: List[ProcessedDatabase]
    pirParameter: IndexPirParameter
    keywordPirParameter: KeywordPirParameter
    table: Optional[CuckooTable]  # None for a database loaded from its serialization
    symmetricPirConfig: Optional[SymmetricPirConfig] = None  # as ProcessedDatabaseWithParameters keeps it

    def save(self, path) -> None:
        """The shard's ProcessedDatabase.save(to:) (KeywordPirProtocol.swift:230-239): the tables' plaintexts
        concatenated in table order, serialized on the device."""
        _save_databases(self.databases, path)

    @staticmethod
    def load(path, context: Context, pirParameter: IndexPirParameter, keywordPirParameter: KeywordPirParameter,
             symmetricPirConfig: Optional[SymmetricPirConfig] = None) -> "ProcessedKeywordDatabase":
        """A saved shard (ProcessedDatabase(from:context:)) cut into hashFunctionCount tables as
        KeywordPirServer.init(context:processed:) does (KeywordPirProtocol.swift:161-171), without its cuckoo table.
        The parameters are the caller's: the reference keeps them in a separate protobuf file."""
        databases = ProcessedDatabase.load(context, path, keywordPirParameter.hashFunctionCount)
        return ProcessedKeywordDatabase(databases, pirParameter, keywordPirParameter, None, symmetricPirConfig)

    def close(self):
        for db in self.databases:
            db.close()
        if self.table is not None:
            self.table.close()


class KeywordPirClient:
    """KeywordPirClient<MulPirClient> (KeywordPirProtocol.swift:280-392), on the device."""

    def __init__(self, keywordParameter: KeywordPirParameter, pirParameter: IndexPirParameter, context: Context):
        self.keywordParameter, self.context = keywordParameter, context
        self.indexPirClient = MulPirClient(pirParameter, context)

    def _indices(self, keyword: bytes) -> List[int]:
        return HashKeyword.hashIndices(bytes(keyword), self.indexPirClient.parameter.entryCount,
                                       self.keywordParameter.hashFunctionCount)

    def generateEvaluationKey(self, secretKey: SecretKey) -> EvaluationKey:
        return self.indexPirClient.generateEvaluationKey(secretKey)

    def generateQuery(self, keyword: bytes, secretKey: SecretKey) -> np.ndarray:
        """KeywordPirClient.generateQuery (:326-334): an index query at the keyword's hashIndices, one per table."""
        return self.indexPirClient.generateQuery(self._indices(keyword), secretKey)

    def decrypt(self, response, keyword: bytes, secretKey: SecretKey) -> Optional[bytes]:
        """KeywordPirClient.decrypt (:343-359): the value stored with the keyword in one of its buckets, or None."""
        keyword_hash = int(HashKeyword.hashes([bytes(keyword)])[0])
        for raw in self.indexPirClient.decrypt(response, self._indices(keyword), secretKey):
            value = HashBucket.find(HashBucket.deserialize(raw), keyword_hash)
            if value is not None:
                return value
        return None

    def queryMessage(self, keyword: bytes, secretKey: SecretKey) -> bytes:
        """generateQuery as a pir.v1.EncryptedIndices message (MulPirClient.queryMessage at the keyword's hashIndices)."""
        return self.indexPirClient.queryMessage(self._indices(keyword), secretKey)

    def evaluationKeyMessage(self, secretKey: SecretKey):
        """(key, SerializedEvaluationKey message) as MulPirClient.evaluationKeyMessage."""
        return self.indexPirClient.evaluationKeyMessage(secretKey)

    def decryptResponseMessage(self, message: bytes, keyword: bytes, secretKey: SecretKey) -> Optional[bytes]:
        """decrypt of an api.pir.v1.PIRResponse of hashFunctionCount replies."""
        response = responseFromMessage(self.context, message, self.keywordParameter.hashFunctionCount,
                                       self.indexPirClient.parameter)
        return self.decrypt(response, keyword, secretKey)

    def countEntriesInResponse(self, response, secretKey: SecretKey) -> int:
        """KeywordPirClient.countEntriesInResponse (:376-391): the slots of every bucket found in the replies' bytes."""
        found = 0
        for data in self.indexPirClient.decryptFull(response, secretKey):
            offset = 0
            while offset < len(data):
                try:
                    slots = HashBucket.deserialize(data[offset:])
                except PirError:
                    break
                found += len(slots)
                offset += HashBucket.serializedSize(slots)
        return found

    def noiseBudget(self, response, secretKey: SecretKey) -> float:
        return self.indexPirClient.noiseBudget(response, secretKey)


class KeywordPirServer:
    """KeywordPirServer<MulPirServer> (KeywordPirProtocol.swift:137-276)."""

    def __init__(self, context: Context, processed: ProcessedKeywordDatabase):
        self.context, self.processed = context, processed
        self.hashFunctionCount = processed.keywordPirParameter.hashFunctionCount
        self.indexPirServer = MulPirServer(processed.pirParameter, context, processed.databases)

    @property
    def indexPirParameter(self) -> IndexPirParameter:
        return self.processed.pirParameter

    @staticmethod
    def processOnDevice(database: Sequence[KeywordValuePair], config: KeywordPirConfig, context: Context,
                        rng: Rng = Rng.splitMix64(),
                        symmetricPirConfig: Optional[SymmetricPirConfig] = None) -> ProcessedKeywordDatabase:
        """KeywordPirServer.process (KeywordPirProtocol.swift:191-247): the cuckoo table, its IndexPirParameter
        (entryCount = bucketsPerTable, batchSize = hashFunctionCount, no entry-size encoding) and one MulPir database per
        table, built from the serialized buckets without them leaving the device.  The database is taken as given: a
        symmetric PIR database is one KeywordDatabase.symmetricPIRProcess has already processed, and symmetricPirConfig
        is only stored with the result."""
        cuckoo = config.cuckooTableConfig
        table = CuckooTable(context, cuckoo, database, rng)
        try:
            if config.useMaxSerializedBucketSize or isinstance(cuckoo.bucketCount, FixedSize):
                entry_size = cuckoo.maxSerializedBucketSize
            else:
                entry_size = table.maxSerializedBucketSize()
            parameter = MulPir.generateParameter(
                IndexPirConfig(table.bucketsPerTable, entry_size, config.dimensionCount, cuckoo.hashFunctionCount,
                               config.unevenDimensions, config.keyCompression, False), context)
            tables = cuckoo.tableCount
            handles = (C.c_void_p * tables)()
            dims = (C.c_int32 * len(parameter.dimensions))(*parameter.dimensions)
            _check(load_library().hecuda_keyword_pir_databases_create(context._h, table._h, entry_size, dims, len(dims),
                                                                      handles))
        except Exception:
            table.close()
            raise
        count = -(-parameter.encodedEntrySize // bytesPerPlaintext(context)) * int(np.prod(parameter.dimensions))
        databases = [ProcessedDatabase._adopt(context, C.c_void_p(h), count) for h in handles]
        return ProcessedKeywordDatabase(databases, parameter, config.parameter, table, symmetricPirConfig)

    def computeResponse(self, query, evaluationKey: EvaluationKey) -> np.ndarray:
        """computeResponse(to:using:): MulPir over the hashFunctionCount tables with indicesCount = hashFunctionCount.
        Returns (hashFunctionCount, chunkCount, 2, 1, N)."""
        return self.indexPirServer.computeResponse(query, evaluationKey, indicesCount=self.hashFunctionCount)

    def computeResponses(self, queries, evaluationKeys: Sequence[EvaluationKey]) -> np.ndarray:
        """computeResponse for many clients in one call; client c's reply equals computeResponse(queries[c], keys[c])."""
        return self.indexPirServer.computeResponses(queries, evaluationKeys, indicesCount=self.hashFunctionCount)

    def computeResponseWire(self, queryPoly0, querySeeds, evaluationKey: EvaluationKey):
        """Serialized seeded query in, serialized reply out (PirWire.computeResponse)."""
        return PirWire.computeResponse(self.indexPirServer, queryPoly0, querySeeds, evaluationKey, self.hashFunctionCount)

    def computeResponsesWire(self, queryPoly0, querySeeds, evaluationKeys: Sequence[EvaluationKey]):
        return PirWire.computeResponses(self.indexPirServer, queryPoly0, querySeeds, evaluationKeys, self.hashFunctionCount)

    def computeResponsesProto(self, messages: Sequence[bytes], evaluationKeys: Sequence[EvaluationKey]) -> List[bytes]:
        """One EncryptedIndices message per client in, one PIRResponse per client out, with indicesCount =
        hashFunctionCount (PirWire.computeResponsesProto)."""
        return PirWire.computeResponsesProto(self.indexPirServer, messages, evaluationKeys, self.hashFunctionCount)

    def validate(self, row: KeywordValuePair, trials: int = 1) -> ShardValidationResult:
        """KeywordDatabase.validateShard (KeywordDatabase.swift:557-630): row = (keyword, value).  Every step runs on the
        device; raises PirError("Insufficient noise budget") or PirError("Incorrect PIR response") when a trial's reply
        does not decrypt to the value."""
        keyword, value = bytes(row[0]), bytes(row[1])
        client = KeywordPirClient(self.processed.keywordPirParameter, self.indexPirParameter, self.context)
        return _validate(trials, client, self.computeResponse, lambda sk: client.generateQuery(keyword, sk),
                         lambda response, sk: client.decrypt(response, keyword, sk), value, client.countEntriesInResponse)
