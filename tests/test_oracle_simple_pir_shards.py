"""Sharding on the host: hecuda.simple_pir's DatabaseMap / ShardMap against the reference's shardMapTest and against
tests/simple_pir_shards_ref.py, and the all-shards client (tests/simple_pir_shards_ref.py over the oracle's Client)
round-tripping through the oracle's server."""
import numpy as np
import pytest

import simple_pir_shards_ref as ref
from hecuda import simple_pir as sp
from oracle import simple_pir_oracle as osp


def test_shard_map_of_the_reference():
    """shardMapTest: 1000 entries of 100..999 bytes, 5 shards, chunk 256."""
    rng = np.random.default_rng(1)
    entries = [(i, rng.integers(0, 256, size=int(rng.integers(100, 1000)), dtype=np.uint8).tobytes()) for i in range(1000)]
    database_map, shards = sp.DatabaseMap.shardDatabase(entries, 5, 256, rng=rng)
    mapping = sp.ShardMap(database_map)
    assert mapping.shardCount == 5
    assert mapping.chunkSize == 256
    assert mapping.maximumChunkCount == -(-1000 // 256) == 4
    assert len(mapping.mapping) == 1000
    assert mapping.chunksPerShard == 1
    assert sum(len(s) for s in shards) == sum(len(e.chunks) for e in database_map.entries)


@pytest.mark.parametrize("matrix", [False, True])
def test_database_map_matches_the_restatement_under_one_rng(matrix):
    rng = np.random.default_rng(7)
    if matrix:
        raw = rng.integers(0, 256, size=(300, 50), dtype=np.uint8)
        entries = [(i, raw[i].tobytes()) for i in range(300)]
    else:
        entries = [(1000 + i, rng.integers(0, 256, size=int(rng.integers(0, 90)), dtype=np.uint8).tobytes())
                   for i in range(300)]
    shard_count, chunk_size = 3, 15
    database_map, shards = sp.DatabaseMap.shardDatabase(raw if matrix else entries, shard_count, chunk_size,
                                                        rng=np.random.default_rng(11))
    perms = np.random.default_rng(11).permuted(np.tile(np.arange(shard_count), (len(entries), 1)), axis=1)
    mapped, expect = ref.shard_database(entries, shard_count, chunk_size, perms)
    got = [(e.originalIndex, e.size, [(c.shardIndex, c.index) for c in e.chunks]) for e in database_map.entries]
    assert got == mapped
    assert all(np.array_equal(a, b) for a, b in zip(shards, expect))


def test_all_shards_client_round_trip_over_the_oracle_server():
    rng = np.random.default_rng(3)
    pt, ct, n, chunk_size, shard_count = 14, 42, 1024, 15, 2
    entries = [(i, rng.integers(0, 256, size=50, dtype=np.uint8).tobytes()) for i in range(40)]
    perms = [rng.permutation(shard_count) for _ in entries]
    mapped, shards = ref.shard_database(entries, shard_count, chunk_size, perms)
    servers, clients = [], []
    for s, rows in enumerate(shards):
        prm = osp.computing_params(pt, len(rows), chunk_size)
        db = osp.process_database(rows, pt, prm["entries_per_column"], prm["chunks_per_entry"], prm["database_columns"])
        seed = bytes([s]) * 32
        hint = osp.hint(db, seed, n, osp.ntt_friendly_mod(ct, n))
        servers.append(db)
        clients.append(osp.Client(dict(prm, N=n, pt=pt, ct=ct, entry_size=chunk_size), hint, seed, rng))
    client = ref.ClientForAllShards(mapped, chunk_size, clients)
    for index in (0, 17, 39, 140):
        queries = client.query(index)
        assert len({len(q) for q in queries}) == 1
        responses = [[osp.response(db, q[1][0], ct) for q in qs] for db, qs in zip(servers, queries)]
        got = client.decrypt(responses, queries, index)
        assert got == (entries[index][1] if index < 40 else None)
