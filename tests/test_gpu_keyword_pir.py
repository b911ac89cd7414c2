"""Keyword PIR on the GPU: keyword hashes, candidate indices and bucket serialization on the device, the cuckoo
placement through the C ABI, one resident MulPir database per table, and keyword queries answered end to end.

The oracle (oracle/keyword_oracle.py, pinned on the reference's HashBucketTests and CuckooTableTests) is the reference
for every byte; the databases must equal hecuda_pir_database_create_from_entries on the oracle's bucket bytes."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import keyword_pir as kw
from hecuda import pir
from oracle import keyword_oracle as K
from oracle import oracle as orc
from oracle import pir_oracle as opir
from test_gpu_evk_wire import read_device
from test_keyword_pir_emulation import CASES, mixed_rows

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:346-367)
ERR_INVALID_ARGUMENT = -1


@pytest.fixture(scope="module")
def g():
    ctx = hecuda.Context(4096, PIR_MODULI, 17)
    yield ctx
    ctx.close()


def device_config(config: K.CuckooTableConfig) -> kw.CuckooTableConfig:
    bucket = (kw.AllowExpansion(config.expansion_factor, config.target_load_factor) if config.bucket_count is None
              else kw.FixedSize(config.bucket_count))
    return kw.CuckooTableConfig(config.hash_function_count, config.max_eviction_count, config.max_serialized_bucket_size,
                                bucket, config.multiple_tables, config.slot_count)


def test_device_hashes_and_indices_match_the_oracle():
    rng = random.Random(1)
    keywords = [bytes(rng.randrange(256) for _ in range(rng.randint(0, 130))) for _ in range(10000)]
    hashes = kw.HashKeyword.hashes(keywords)
    assert [int(h) for h in hashes] == [K.keyword_hash(k) for k in keywords]
    for buckets, h in ((8, 3), (2048, 5), (1000003, 2), (3, 3)):
        got = kw.HashKeyword.hashIndicesOfHashes(hashes[:2000], buckets, h)
        want = [K.hash_indices_of_hash(int(x), buckets, h) for x in hashes[:2000]]
        assert got.tolist() == want
    # HashBucketTests.hashIndices (:75-79)
    assert kw.HashKeyword.hashIndices(bytes([0, 1, 2, 3]), 8, 3) == [7, 3, 0]
    assert kw.HashKeyword.hashIndices(bytes([3, 2, 1, 0]), 2048, 5) == [1989, 1767, 1260, 242, 1122]


def test_summarize_kat(g):
    # CuckooTableTests.summarize (:69-90)
    rng = K.TestRng(1)
    rows = K.random_keyword_pir_database(100, 10, rng)
    config = kw.CuckooTableConfig(2, 100, 50, kw.AllowExpansion(1.1, 0.9))
    table = kw.CuckooTable(g, config, rows, kw.Rng.counter(rng.counter))
    info = table.summarize()
    assert (info.entryCount, info.bucketCount, info.emptyBucketCount) == (100, 80, 19)
    assert info.loadFactor == np.float32(0.52)
    table.close()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("rng_kind", [0, 1])
def test_serialized_buckets_match_the_oracle(g, case, rng_kind):
    config, rows, seed = CASES[case]()
    expected = K.CuckooTable(config, rows, K.TestRng(seed) if rng_kind == 0 else K.SplitMix64(seed))
    table = kw.CuckooTable(g, device_config(config), rows, kw.Rng(rng_kind, seed))
    assert table.serializeBuckets() == expected.serialize_buckets()
    assert table.bucketsPerTable == expected.buckets_per_table
    assert table.maxSerializedBucketSize() == expected.max_serialized_bucket_size()
    assert table.summarize().emptyBucketCount == expected.summarize()["emptyBucketCount"]
    table.close()


def keyword_setup(g, rows, config, dims, rng=kw.Rng.counter(3)):
    kconfig = kw.KeywordPirConfig(dims, config, False, "noCompression")
    return kw.KeywordPirServer.processOnDevice(rows, kconfig, g, rng)


@pytest.mark.parametrize("dims", [1, 2])
@pytest.mark.parametrize("shape", ["fixed_values", "mixed"])
def test_databases_equal_create_from_entries(g, dims, shape):
    rows = (K.random_keyword_pir_database(500, 40, K.TestRng(2)) if shape == "fixed_values"
            else mixed_rows(3, 100))
    config = kw.CuckooTableConfig.defaultKeywordPir(200) if shape == "fixed_values" else \
        kw.CuckooTableConfig(2, 100, 100, kw.AllowExpansion(1.1, 0.9))
    processed = keyword_setup(g, rows, config, dims)
    buckets = processed.table.serializeBuckets()
    per = processed.table.bucketsPerTable
    assert len(processed.databases) == 2
    for t, db in enumerate(processed.databases):
        reference = pir.MulPirServer.processOnDevice(buckets[t * per:(t + 1) * per], g, processed.pirParameter)
        assert db.count == reference.count
        assert np.array_equal(read_device(*db.deviceBuffer()), read_device(*reference.deviceBuffer()))
        assert np.array_equal(db.presentFlags(), reference.presentFlags())
        reference.close()
    processed.close()


@pytest.mark.parametrize("dims", [1, 2])
def test_keyword_queries_end_to_end(g, dims):
    o = orc.Context(4096, PIR_MODULI, 17)
    rows = mixed_rows(3, 100)  # reaches the branch where the reference loses a row
    config = kw.CuckooTableConfig(2, 100, 100, kw.AllowExpansion(1.1, 0.9))
    processed = keyword_setup(g, rows, config, dims, kw.Rng.counter(10))
    server = kw.KeywordPirServer(g, processed)
    param, h = processed.pirParameter, 2
    oparam = opir.generate_parameter(opir.IndexPirConfig(param.entryCount, param.entrySizeInBytes, dims, h, False,
                                                         "noCompression", False), o.n, o.t)
    assert oparam.dimensions == param.dimensions
    # the oracle-processed tables
    otable = K.CuckooTable(K.CuckooTableConfig(2, 100, 100), rows, K.TestRng(10))
    assert otable.summarize()["entryCount"] == len(rows)
    _, odbs, entry_size = K.process(o, otable, dims)
    assert entry_size == param.entrySizeInBytes
    absent = [b"absent keyword %d" % i for i in range(2)]
    lookups = [rows[0][0], rows[57][0], rows[-1][0], absent[0]], [rows[20][0], absent[1], rows[99][0], rows[5][0]]
    keys, queries, secrets = [], [], []
    for c, words in enumerate(lookups):
        sk, relin = o.keygen(100 + c)
        key = hecuda.EvaluationKey(g, relin)
        okeys = {}
        for i, e in enumerate(param.evaluationKeyConfig.galoisElements):
            okeys[e] = o.galois_keygen(7000 + 31 * c + i, sk, e)
            key.setGaloisKey(e, okeys[e])
        keys.append((key, okeys, relin))
        secrets.append(sk)
        queries.append([np.stack(K.generate_query(o, oparam, w, h, sk, 9000 + 17 * c + j)) for j, w in enumerate(words)])
    values = dict(rows)
    for j in range(len(lookups[0])):
        batch = np.stack([queries[c][j] for c in range(len(lookups))])
        many = server.computeResponses(batch, [k[0] for k in keys])
        for c, words in enumerate(lookups):
            single = server.computeResponse(queries[c][j], keys[c][0])
            assert np.array_equal(many[c], single)
            reply = [[single[qi, chunk] for chunk in range(single.shape[1])] for qi in range(h)]
            assert K.decrypt(o, oparam, reply, words[j], h, secrets[c]) == values.get(words[j])
            if c == 0 and j < 2:  # bit-identical to the oracle's response on the oracle's tables
                expected = opir.compute_response(o, list(queries[c][j]), h, keys[c][1], keys[c][2], odbs, oparam)
                for qi in range(h):
                    for chunk in range(single.shape[1]):
                        assert np.array_equal(single[qi, chunk], expected[qi][chunk])
    for key, _, _ in keys:
        key.close()
    processed.close()


def _raw_table(g, rows, config, rng=0):
    keywords, koff = kw._concatenate([k for k, _ in rows])
    values, voff = kw._concatenate([v for _, v in rows])
    h = C.c_void_p(1234)
    rc = hecuda.load_library().hecuda_cuckoo_table_create(g._h, hecuda._ptr(keywords), hecuda._ptr(koff), hecuda._ptr(values),
                                                          hecuda._ptr(voff), len(rows), C.byref(config), rng, 0, C.byref(h))
    return rc, h


def test_errors_leave_nothing_allocated(g):
    import torch
    lib = hecuda.load_library()
    rows = K.random_keyword_pir_database(2000, 10, K.TestRng(0))
    good = kw.CuckooTableConfig(2, 100, 50, kw.AllowExpansion(1.1, 0.9))._c()
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        for field, value, message in (("hash_function_count", 0, "invalidCuckooConfig"),
                                      ("max_serialized_bucket_size", 10, "invalidCuckooConfig"),
                                      ("slot_count", 256, "invalidCuckooConfig"),
                                      ("expansion_factor", 1.0, "invalidCuckooConfig"),
                                      ("target_load_factor", 0.0, "invalidCuckooConfig"),
                                      ("max_eviction_count", 0, "invalidCuckooConfig"),
                                      ("fixed_bucket_count", 10, "failedToConstructCuckooTable")):
            cfg = kw._Config.from_buffer_copy(good)
            setattr(cfg, field, value)
            rc, h = _raw_table(g, rows, cfg)
            assert rc == ERR_INVALID_ARGUMENT and h.value is None, field
            assert message in lib.hecuda_last_error().decode(), field
        rc, h = _raw_table(g, rows, good, rng=7)
        assert rc == ERR_INVALID_ARGUMENT and h.value is None
        big = kw.CuckooTableConfig(2, 100, 1 << 20, kw.AllowExpansion(1.1, 0.9))._c()
        rc, h = _raw_table(g, [(b"k", bytes(65536))], big)
        assert rc == ERR_INVALID_ARGUMENT and h.value is None
        assert "invalidHashBucketEntryValueSize" in lib.hecuda_last_error().decode()
        rc, h = _raw_table(g, [(b"k", bytes(40))], good)
        assert rc == ERR_INVALID_ARGUMENT and "failedToConstructCuckooTable" in lib.hecuda_last_error().decode()
        # keyword PIR needs one table per hash function
        single = kw.CuckooTable(g, kw.CuckooTableConfig(2, 100, 50, kw.AllowExpansion(1.1, 0.9), multipleTables=False),
                                rows[:100])
        out = (C.c_void_p * 2)(5, 6)
        dims = (C.c_int32 * 1)(single.bucketsPerTable)
        assert lib.hecuda_keyword_pir_databases_create(g._h, single._h, 50, dims, 1, out) == ERR_INVALID_ARGUMENT
        assert "invalidCuckooConfig" in lib.hecuda_last_error().decode()
        assert out[0] is None  # one table
        single.close()
        out[0], out[1] = 5, 6
        # an entry size below the largest bucket
        table = kw.CuckooTable(g, kw.CuckooTableConfig(2, 100, 50, kw.AllowExpansion(1.1, 0.9)), rows[:100])
        dims = (C.c_int32 * 1)(table.bucketsPerTable)
        assert lib.hecuda_keyword_pir_databases_create(g._h, table._h, 12, dims, 1, out) == ERR_INVALID_ARGUMENT
        assert "invalidDatabaseEntrySize" in lib.hecuda_last_error().decode()
        assert out[0] is None and out[1] is None
        table.close()
    with pytest.raises(pir.PirError, match="invalidCuckooConfig"):
        kw.KeywordPirConfig(1, kw.CuckooTableConfig(2, 100, 50, kw.AllowExpansion(1.1, 0.9), multipleTables=False), False,
                            "noCompression")
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 64 << 20


def test_keyword_database_shards_by_device_hash():
    rows = K.random_keyword_pir_database(300, 4, K.TestRng(0))
    database = kw.KeywordDatabase(rows, kw.Sharding.shardCount(5))
    for sid, shard in database.shards.items():
        for keyword, _ in shard:
            assert K.shard_index(keyword, 5) == int(sid)
    assert sum(len(s) for s in database.shards.values()) == 300
    double = kw.KeywordDatabase(rows, kw.Sharding.shardCount(3), kw.ShardingFunction.doubleMod(7))
    for sid, shard in double.shards.items():
        for keyword, _ in shard:
            assert K.keyword_hash(keyword) % 7 % 3 == int(sid)
    with pytest.raises(pir.PirError, match="invalidDatabaseDuplicateKeyword"):
        kw.KeywordDatabase(rows + [(rows[3][0], b"other")], kw.Sharding.shardCount(5))
