"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's keyword PIR (hashlib for SHA-256).

Only tests/ and tools/ may import this module; the product (swift-homomorphic-encryption_b200/) never does.

Every function names the reference code it follows (paths relative to Sources/PrivateInformationRetrieval/):

  * HashKeyword        KeywordPir/HashBucket.swift:208-270
  * HashBucket         KeywordPir/HashBucket.swift:18-206
  * CuckooTable        KeywordPir/CuckooTable.swift
  * process            KeywordPir/KeywordPirProtocol.swift:191-247 (through pir_oracle.process_database)
  * client             KeywordPir/KeywordPirProtocol.swift:326-359 (through pir_oracle.generate_query / decrypt_response)
  * test databases     _TestUtilities/PirUtilities/PirTestUtils.swift:79-112 with RandomNumberGenerator.fill
                       (HomomorphicEncryption/Random/PseudoRandomNumberGenerator.swift:64-88)

Pinned on the reference's HashBucketTests and CuckooTableTests (tests/test_oracle_keyword.py).

One deliberate divergence, shared with the library (csrc/cuckoo.hpp): when no candidate bucket has a swap index,
CuckooTable.insertLoop expands the table and returns without inserting the pair in hand (CuckooTable.swift:455-457), so
that row is lost.  Here the pair is inserted again after the expansion, as the branch at :402-406 does; `lose_rows=True`
restores the reference's behaviour.
"""
from __future__ import annotations

import hashlib
import math
import struct
from dataclasses import dataclass

from . import pir_oracle as P

MAX_RETRIES = 10
MAX_SLOT_COUNT = 255
MAX_VALUE_SIZE = 0xFFFF
MASK64 = (1 << 64) - 1


class PirError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ HashKeyword
def keyword_hash(keyword: bytes) -> int:
    """HashKeyword.hash: the first 8 bytes of SHA-256(keyword) as a little-endian UInt64."""
    return int.from_bytes(hashlib.sha256(bytes(keyword)).digest()[:8], "little")


def index_from_hash(keyword_hash_value: int, bucket_count: int, counter: int) -> int:
    """HashKeyword.indexFromHash: SHA-256(bigEndian(hash) || UInt8(counter)), first 8 bytes LE, mod bucketCount."""
    digest = hashlib.sha256(struct.pack(">Q", keyword_hash_value) + bytes([counter])).digest()
    return int.from_bytes(digest[:8], "little") % bucket_count


def hash_indices_of_hash(h: int, bucket_count: int, hash_function_count: int) -> list:
    candidates = []
    for _ in range(hash_function_count):
        counter = 0
        index = index_from_hash(h, bucket_count, counter)
        while index in candidates and counter < MAX_RETRIES:
            counter += 1
            index = index_from_hash(h, bucket_count, counter)
        candidates.append(index)
    return candidates


def hash_indices(keyword: bytes, bucket_count: int, hash_function_count: int) -> list:
    """HashKeyword.hashIndices (HashBucket.swift:221-235)."""
    return hash_indices_of_hash(keyword_hash(keyword), bucket_count, hash_function_count)


def shard_index(keyword: bytes, shard_count: int) -> int:
    """Keyword.shardIndex (KeywordDatabase.swift:56-62)."""
    return keyword_hash(keyword) % shard_count


# ------------------------------------------------------------------------------------------------ HashBucket
def serialized_size(values) -> int:
    """HashBucket.serializedSize(values:): slot count byte + (8 + 2 + len) per value."""
    return 1 + sum(10 + len(v) for v in values)


def serialized_size_single(value_size: int) -> int:
    return 11 + value_size


def serialize_bucket(slots) -> bytes:
    """HashBucket.serialize: slots = [(keyword hash, value)]."""
    if len(slots) > MAX_SLOT_COUNT:
        raise PirError(f"invalidHashBucketSlotCount(maxCount: {MAX_SLOT_COUNT})")
    out = bytearray([len(slots)])
    for h, value in slots:
        if len(value) > MAX_VALUE_SIZE:
            raise PirError(f"invalidHashBucketEntryValueSize(maxSize: {MAX_VALUE_SIZE})")
        out += struct.pack("<QH", h, len(value)) + bytes(value)
    return bytes(out)


def deserialize_bucket(raw: bytes) -> list:
    """HashBucket.init(deserialize:) -> [(keyword hash, value)]."""
    if not raw:
        raise PirError("corruptedData: Serialized HashBucket shouldn't be empty.")
    count, offset, slots = raw[0], 1, []
    for _ in range(count):
        if len(raw) < offset + 10:
            raise PirError("corruptedData: Serialized HashBucketEntry should at least have a keyword hash and a value size.")
        h, size = struct.unpack_from("<QH", raw, offset)
        offset += 10
        if offset + size > len(raw):
            raise PirError("corruptedData: HashBucketEntry buffer has less data than expected")
        slots.append((h, bytes(raw[offset:offset + size])))
        offset += size
    return slots


def bucket_find(slots, keyword: bytes):
    """HashBucket.find(keyword:)."""
    h = keyword_hash(keyword)
    for slot_hash, value in slots:
        if slot_hash == h:
            return value
    return None


# ------------------------------------------------------------------------------------------------ generators
class TestRng:
    """_TestUtilities TestRng: next() returns the counter, then adds 1 (wrapping)."""

    def __init__(self, counter: int = 0):
        self.counter = counter & MASK64

    def next(self) -> int:
        value = self.counter
        self.counter = (self.counter + 1) & MASK64
        return value


class SplitMix64:
    def __init__(self, seed: int = 0):
        self.state = seed & MASK64

    def next(self) -> int:
        self.state = (self.state + 0x9E3779B97F4A7C15) & MASK64
        z = self.state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)


def next_upper_bound(rng, n: int) -> int:
    """RandomNumberGenerator.next(upperBound:) (Swift stdlib), which Int.random(in: 0..<n) and randomElement reach."""
    m = rng.next() * n
    if (m & MASK64) < n:
        t = ((1 << 64) - n) % n
        while (m & MASK64) < t:
            m = rng.next() * n
    return m >> 64


def fill(rng, size: int) -> bytes:
    """RandomNumberGenerator.fill: whole little-endian words, then the low bytes of one more."""
    out = bytearray()
    for _ in range(size // 8):
        out += rng.next().to_bytes(8, "little")
    if size % 8:
        out += rng.next().to_bytes(8, "little")[:size % 8]
    return bytes(out)


def random_keyword_pir_database(row_count: int, value_size: int, rng, keyword_size: int = 30) -> list:
    """PirTestUtils.randomKeywordPirDatabase(rowCount:valueSize:using:keywordSize:) -> [(keyword, value)]."""
    seen, rows = set(), []
    while len(rows) < row_count:
        keyword = fill(rng, keyword_size)
        if keyword in seen:
            continue
        seen.add(keyword)
        rows.append((keyword, fill(rng, value_size)))
    return rows


# ------------------------------------------------------------------------------------------------ CuckooTable
@dataclass
class CuckooTableConfig:
    """CuckooTableConfig (CuckooTable.swift:19-157); bucket_count None = .allowExpansion."""

    hash_function_count: int
    max_eviction_count: int
    max_serialized_bucket_size: int
    expansion_factor: float = 1.1
    target_load_factor: float = 0.9
    bucket_count: int | None = None
    multiple_tables: bool = True
    slot_count: int = MAX_SLOT_COUNT

    def __post_init__(self):
        ok = (self.hash_function_count > 0 and self.max_serialized_bucket_size >= serialized_size_single(0)
              and 0 < self.slot_count <= MAX_SLOT_COUNT)
        if self.bucket_count is None:
            ok = ok and self.expansion_factor > 1.0 and self.target_load_factor < 1.0
        else:
            ok = ok and self.max_serialized_bucket_size > 0 and self.bucket_count > 0
        if not ok:
            raise PirError("invalidCuckooConfig")

    @staticmethod
    def default_keyword_pir(max_serialized_bucket_size: int) -> "CuckooTableConfig":
        return CuckooTableConfig(2, 100, max_serialized_bucket_size, 1.1, 0.9)

    def freezing_table_size(self, max_serialized_bucket_size: int, bucket_count: int) -> "CuckooTableConfig":
        """freezingTableSize: fixed size, the default slot count (the reference drops slotCount here)."""
        return CuckooTableConfig(self.hash_function_count, self.max_eviction_count, max_serialized_bucket_size,
                                 bucket_count=bucket_count, multiple_tables=self.multiple_tables)

    @property
    def table_count(self) -> int:
        return self.hash_function_count if self.multiple_tables else 1


def _next_multiple(x: int, m: int) -> int:
    return -(-x // m) * m


class CuckooTable:
    """CuckooTable (CuckooTable.swift:256-505); rows = [(keyword, value)] inserted in order."""

    def __init__(self, config: CuckooTableConfig, rows, rng, lose_rows: bool = False):
        self.config, self.rng, self.lose_rows = config, rng, lose_rows
        self.rows = [(bytes(k), bytes(v)) for k, v in rows]
        self.hashes = [keyword_hash(k) for k, _ in self.rows]
        self._indices = {}
        if config.bucket_count is None:
            minimum = -(-serialized_size([v for _, v in self.rows]) // config.max_serialized_bucket_size)
            target = _next_multiple(int(math.ceil(float(minimum) / config.target_load_factor)), config.table_count)
        else:
            target = _next_multiple(config.bucket_count, config.table_count)
        self.buckets = [[] for _ in range(target)]  # entry ids in slot order
        for e in range(len(self.rows)):
            self.insert(e)

    @property
    def buckets_per_table(self) -> int:
        return len(self.buckets) // self.config.table_count

    def index(self, table: int, i: int) -> int:
        return i if self.config.table_count == 1 else table * self.buckets_per_table + i

    def _candidates(self, e: int) -> list:
        key = (e, self.buckets_per_table)
        if key not in self._indices:
            self._indices[key] = hash_indices_of_hash(self.hashes[e], self.buckets_per_table, self.config.hash_function_count)
        return self._indices[key]

    def _size(self, bucket) -> int:
        return serialized_size([self.rows[e][1] for e in bucket])

    def insert(self, e: int):
        if serialized_size_single(len(self.rows[e][1])) > self.config.max_serialized_bucket_size:
            raise PirError("failedToConstructCuckooTable: value larger than maxSerializedBucketSize allows")
        self.insert_loop(e, self.config.max_eviction_count)

    def insert_loop(self, e: int, remaining: int):
        cfg = self.config
        while True:
            if remaining == 0:
                if cfg.bucket_count is not None:
                    raise PirError("failedToConstructCuckooTable: unable to insert")
                self.expand()
                self.insert(e)
            cand = self._candidates(e)
            keyword, value = self.rows[e]
            for t, i in enumerate(cand):
                if any(self.rows[o][0] == keyword for o in self.buckets[self.index(t, i)]):
                    return
            for t, i in enumerate(cand):  # CuckooBucket.canInsert
                bucket = self.buckets[self.index(t, i)]
                if (len(bucket) < cfg.slot_count
                        and self._size(bucket) + 10 + len(value) <= cfg.max_serialized_bucket_size):
                    bucket.append(e)
                    return
            swaps = []
            for t, i in enumerate(cand):  # CuckooBucket.swapIndices
                at = self.index(t, i)
                bucket = self.buckets[at]
                values = [self.rows[o][1] for o in bucket]
                concatenated = values + [value] + values
                for s in range(len(values)):
                    if serialized_size(concatenated[s + 1:s + 1 + len(values)]) <= cfg.max_serialized_bucket_size:
                        swaps.append((at, s))
            if not swaps:
                self.expand()
                if not self.lose_rows:
                    self.insert(e)
                return
            at, s = swaps[next_upper_bound(self.rng, len(swaps))]
            e, self.buckets[at][s] = self.buckets[at][s], e
            remaining -= 1

    def expand(self):
        cfg = self.config
        if cfg.bucket_count is not None:
            raise PirError("failedToConstructCuckooTable: needed to expand a table that doesn't allow expansion")
        old = self.buckets
        count = _next_multiple(int(math.ceil(float(len(old)) * cfg.expansion_factor)), cfg.table_count)
        self.buckets = [[] for _ in range(count)]
        for bucket in old:
            for e in bucket:
                self.insert(e)

    def serialize_buckets(self) -> list:
        return [serialize_bucket([(self.hashes[e], self.rows[e][1]) for e in b]) for b in self.buckets]

    def max_serialized_bucket_size(self) -> int:
        return max((self._size(b) for b in self.buckets), default=0)

    def summarize(self) -> dict:
        import numpy as np
        sizes = [self._size(b) for b in self.buckets]
        return dict(entryCount=sum(len(b) for b in self.buckets), bucketCount=len(self.buckets),
                    emptyBucketCount=sum(1 for b in self.buckets if not b),
                    loadFactor=np.float32(sum(sizes)) / np.float32(len(self.buckets) * self.config.max_serialized_bucket_size))

    def lookup(self, keyword: bytes):
        """CuckooTable subscript (:492-504)."""
        for t, i in enumerate(hash_indices(keyword, self.buckets_per_table, self.config.hash_function_count)):
            for e in self.buckets[self.index(t, i)]:
                if self.rows[e][0] == keyword:
                    return self.rows[e][1]
        return None


# ------------------------------------------------------------------------------------------------ KeywordPirServer
def process(ctx, table: CuckooTable, dimension_count: int, use_max_serialized_bucket_size: bool = False,
            uneven_dimensions: bool = False, key_compression: str = "noCompression"):
    """KeywordPirServer.process (KeywordPirProtocol.swift:191-247) on a built table -> (IndexPirParameter, [database
    per table], entry size)."""
    cfg = table.config
    entries = table.serialize_buckets()
    if use_max_serialized_bucket_size or cfg.bucket_count is not None:
        entry_size = cfg.max_serialized_bucket_size
    else:
        entry_size = max(len(b) for b in entries)
    per = table.buckets_per_table
    param = P.generate_parameter(P.IndexPirConfig(per, entry_size, dimension_count, cfg.hash_function_count,
                                                  uneven_dimensions, key_compression, False), ctx.n, ctx.t)
    dbs = [P.process_database(ctx, param, entries[s:s + per]) for s in range(0, len(entries), per)]
    return param, dbs, entry_size


def generate_query(ctx, param, keyword: bytes, hash_function_count: int, sk, seed: int) -> list:
    """KeywordPirClient.generateQuery (KeywordPirProtocol.swift:326-334)."""
    return P.generate_query(ctx, param, hash_indices(keyword, param.entry_count, hash_function_count), sk, seed)


def decrypt(ctx, param, response, keyword: bytes, hash_function_count: int, sk):
    """KeywordPirClient.decrypt (KeywordPirProtocol.swift:343-359): the value, or None."""
    indices = hash_indices(keyword, param.entry_count, hash_function_count)
    for raw in P.decrypt_response(ctx, param, response, indices, sk):
        value = bucket_find(deserialize_bucket(raw), keyword)
        if value is not None:
            return value
    return None
