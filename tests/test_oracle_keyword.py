"""The keyword-PIR oracle (oracle/keyword_oracle.py) pinned on the reference's HashBucketTests and CuckooTableTests."""
import random

import numpy as np
import pytest

from oracle import keyword_oracle as K

# HashBucketTests.rawBucket (Tests/PrivateInformationRetrievalTests/HashBucketTests.swift:20-24)
RAW_BUCKET = bytes([3, 24, 95, 141, 179, 34, 113, 254, 37, 5, 0, 87, 111, 114, 108, 100, 82, 117, 17, 222, 175, 220, 211,
                    74, 6, 0, 77, 97, 97, 105, 108, 109, 192, 21, 173, 109, 218, 248, 187, 80, 8, 0, 68, 97, 114, 107, 110,
                    101, 115, 115])


def test_hash_indices_kat():
    # HashBucketTests.hashIndices (:75-79)
    assert K.hash_indices(bytes([0, 1, 2, 3]), 8, 3) == [7, 3, 0]
    assert K.hash_indices(bytes([3, 2, 1, 0]), 2048, 5) == [1989, 1767, 1260, 242, 1122]


def test_raw_bucket_kat():
    # HashBucketTests.bucketDeserialization (:82-87)
    slots = K.deserialize_bucket(RAW_BUCKET)
    assert len(slots) == 3
    assert K.bucket_find(slots, b"Hello") == b"World"
    assert K.bucket_find(slots, b"Goodbye") == b"Darkness"
    assert K.bucket_find(slots, b"Absent") is None
    assert K.serialize_bucket(slots) == RAW_BUCKET
    assert K.serialized_size([v for _, v in slots]) == len(RAW_BUCKET)


def test_summarize_kat():
    # CuckooTableTests.summarize (:69-90): the table's generator continues where the database's draws stopped
    rng = K.TestRng(1)
    rows = K.random_keyword_pir_database(100, 10, rng)
    table = K.CuckooTable(K.CuckooTableConfig(2, 100, 50, 1.1, 0.9), rows, K.TestRng(rng.counter))
    summary = table.summarize()
    assert (summary["entryCount"], summary["bucketCount"], summary["emptyBucketCount"]) == (100, 80, 19)
    assert summary["loadFactor"] == np.float32(0.52)
    for keyword, value in rows:
        assert table.lookup(keyword) == value


def test_fixed_size_kat():
    # CuckooTableTests.cuckooTableFixedSize (:111-136)
    rng = K.TestRng(0)
    rows = K.random_keyword_pir_database(100, 10, rng)
    config = K.CuckooTableConfig(2, 100, 50, 1.1, 0.5)
    grown = K.CuckooTable(config, rows, K.TestRng(rng.counter))
    frozen = config.freezing_table_size(grown.max_serialized_bucket_size(), len(grown.buckets))
    table = K.CuckooTable(frozen, rows, K.TestRng(rng.counter))
    assert table.max_serialized_bucket_size() <= 50
    assert len(table.buckets) == len(grown.buckets)


def test_next_upper_bound_is_swift_lemire():
    # next(upperBound:): the high word of r * n, redrawing while the low word is below (2^64 - n) % n
    rng = K.TestRng(0)
    assert [K.next_upper_bound(rng, 3) for _ in range(3)] == [0, 0, 0]   # small counters: the high word is 0
    big = K.TestRng((1 << 64) - 1)
    assert K.next_upper_bound(big, 7) == ((1 << 64) - 1) * 7 >> 64


@pytest.mark.parametrize("kwargs", [dict(hash_function_count=0), dict(max_serialized_bucket_size=10),
                                    dict(slot_count=0), dict(slot_count=256), dict(expansion_factor=1.0),
                                    dict(target_load_factor=1.0)])
def test_config_errors(kwargs):
    args = dict(hash_function_count=2, max_eviction_count=100, max_serialized_bucket_size=50)
    args.update(kwargs)
    with pytest.raises(K.PirError, match="invalidCuckooConfig"):
        K.CuckooTableConfig(**args)
    with pytest.raises(K.PirError, match="invalidCuckooConfig"):
        K.CuckooTableConfig(2, 100, 50, bucket_count=0)


def test_size_errors():
    with pytest.raises(K.PirError, match="failedToConstructCuckooTable"):
        K.CuckooTable(K.CuckooTableConfig(2, 100, 50), [(b"k", bytes(40))], K.TestRng(0))
    with pytest.raises(K.PirError, match="invalidHashBucketEntryValueSize"):
        K.serialize_bucket([(0, bytes(65536))])
    with pytest.raises(K.PirError, match="invalidHashBucketSlotCount"):
        K.serialize_bucket([(0, b"")] * 256)
    rng = K.TestRng(0)
    rows = K.random_keyword_pir_database(100, 10, rng)
    with pytest.raises(K.PirError, match="failedToConstructCuckooTable"):
        K.CuckooTable(K.CuckooTableConfig(2, 100, 50, bucket_count=10), rows, K.TestRng(0))


def mixed_rows(seed, count):
    """12-byte keywords with 0, 1, 2, 30 or 60-byte values."""
    r = random.Random(seed)
    return [(bytes(r.randrange(256) for _ in range(12)), bytes(r.randrange(256) for _ in range(r.choice([0, 1, 2, 30, 60]))))
            for _ in range(count)]


# seed 3, 100 rows, maxSerializedBucketSize 100, h = 2, TestRng(counter: 10): the reference's loop loses one row
DIVERGENT = dict(seed=3, count=100, size=100, counter=10)


def test_divergent_branch_keeps_every_row():
    rows = mixed_rows(DIVERGENT["seed"], DIVERGENT["count"])
    config = K.CuckooTableConfig(2, 100, DIVERGENT["size"])
    reference = K.CuckooTable(config, rows, K.TestRng(DIVERGENT["counter"]), lose_rows=True)
    assert reference.summarize()["entryCount"] == len(rows) - 1
    table = K.CuckooTable(config, rows, K.TestRng(DIVERGENT["counter"]))
    assert table.summarize()["entryCount"] == len(rows)
    for keyword, value in rows:
        assert table.lookup(keyword) == value
        found = [K.bucket_find(K.deserialize_bucket(table.serialize_buckets()[table.index(t, i)]), keyword)
                 for t, i in enumerate(K.hash_indices(keyword, table.buckets_per_table, 2))]
        assert value in found


def test_duplicate_keywords_keep_the_first_row():
    rows = [(b"a", b"1"), (b"b", b"2"), (b"a", b"3")]
    table = K.CuckooTable(K.CuckooTableConfig(2, 100, 50), rows, K.TestRng(0))
    assert table.summarize()["entryCount"] == 2
    assert table.lookup(b"a") == b"1"


def test_splitmix64_is_the_standard_sequence():
    rng = K.SplitMix64(0)
    assert [rng.next() for _ in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
