"""Sharded SimplePIR on the GPU (hecuda.simple_pir.SimplePirShardedServer over csrc/simple_pir.cu): process_shards
bit-exact against the oracle's process_database and hint for every shard of a host shardDatabase, the grouped response
bit-identical to per-shard hecuda_simple_pir_compute_response (ragged shards, full-width words, several client counts,
past the 32 shards of one launch), launches per call, the reference's sharded flows through the all-shards client,
the device-pointer call, save/load, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import hecuda
import simple_pir_shards_ref as ref
from hecuda import simple_pir as sp
from oracle import simple_pir_oracle as osp

pytestmark = pytest.mark.gpu


def enc(pt=14, ct=42, n=16, std=3.2):
    return sp.SimplePirEncryptionParams(pt, ct, n, std, "unchecked")


def variable_entries(rng, count, low, high):
    return [(i, rng.integers(0, 256, size=int(rng.integers(low, high)), dtype=np.uint8).tobytes()) for i in range(count)]


@pytest.mark.parametrize("shards,scalar,shared_seed,equal_sizes", [
    (1, np.uint64, True, True), (2, np.uint32, False, False), (5, np.uint64, False, False), (5, np.uint32, True, True),
    (2, np.uint64, True, False)])
def test_process_shards_is_bit_exact(shards, scalar, shared_seed, equal_sizes):
    rng = np.random.default_rng(shards * 10 + int(shared_seed))
    entries = (rng.integers(0, 256, size=(300, 40), dtype=np.uint8) if equal_sizes else variable_entries(rng, 300, 1, 90))
    seed = bytes(range(32)) if shared_seed else None
    pt, ct = (7, 28) if scalar == np.uint32 else (14, 42)
    server = sp.SimplePirShardedServer.process(entries, enc(pt, ct), shards, chunkSize=None if equal_sizes else 17, seed=seed,
                                               scalar=scalar, rng=np.random.default_rng(5))
    chunk = server.databaseMap.chunkSize
    assert chunk == (-(-40 // shards) if equal_sizes else 17)
    database_map, host_shards = sp.DatabaseMap.shardDatabase(entries, shards, chunk, rng=np.random.default_rng(5))
    assert database_map == server.databaseMap
    p = osp.ntt_friendly_mod(ct, 16)
    seeds = set()
    for s, rows in enumerate(host_shards):
        prm = server.params[s]
        assert prm == sp.SimplePirParameters.computingParams(enc(pt, ct), len(rows), chunk, prm.seed)
        db = osp.process_database(rows, pt, prm.entriesPerColumn, prm.chunksPerEntry, prm.databaseColumns)
        assert np.array_equal(server.databases[s].export().astype(np.uint64), db), s
        assert np.array_equal(server.hints[s].astype(np.uint64), osp.hint(db, prm.seed, 16, p)), s
        seeds.add(prm.seed)
    assert len(seeds) == (1 if shared_seed else shards)


def ragged_server(rng, shapes, scalar, ct=42, pt=14):
    """shapes: (entry bytes, entriesPerColumn, chunksPerEntry, databaseColumns) per shard, random DB' values."""
    dbs, hints, params = [], [], []
    for size, epc, cpe, k in shapes:
        prm = sp.SimplePirParameters(enc(pt, ct), size, epc, cpe, k)
        db = rng.integers(0, 1 << pt, size=(prm.columnSize, k), dtype=np.uint64).astype(scalar)
        dbs.append(sp.SimplePirDatabase.create(db, prm, scalar))
        hints.append(np.zeros((prm.columnSize, 16), scalar))
        params.append(prm)
    return sp.SimplePirShardedServer(dbs, hints, params, scalar)


def random_requests(rng, server, clients, per_shard):
    info = np.iinfo(server.scalar)
    return [[rng.integers(0, int(info.max), size=(per_shard, p.chunksPerEntry, p.databaseColumns), dtype=np.uint64,
                          endpoint=True).astype(server.scalar) for p in server.params] for _ in range(clients)]


def per_shard_responses(server, requests):
    singles = [sp.SimplePirServer(db, h, p, server.scalar) for db, h, p in zip(server.databases, server.hints, server.params)]
    return [[singles[s].computeResponses(q) for s, q in enumerate(client)] for client in requests]


RAGGED = [(2 * 40, 1, 2, 700), (10, 3, 1, 5), (300, 1, 6, 33), (8, 1, 1, 64 * 32 * 3 + 5), (600, 1, 1, 1)]


@pytest.mark.parametrize("clients", [1, 3, 17])
@pytest.mark.parametrize("scalar,ct", [(np.uint32, 31), (np.uint64, 42), (np.uint64, 61)])
def test_grouped_response_equals_per_shard_responses(clients, scalar, ct):
    rng = np.random.default_rng(clients * ct)
    server = ragged_server(rng, RAGGED, scalar, ct=ct)
    requests = random_requests(rng, server, clients, 2)
    got = server.computeResponses(requests)
    expect = per_shard_responses(server, requests)
    for c in range(clients):
        for s in range(len(RAGGED)):
            assert np.array_equal(got[c][s], expect[c][s]), (c, s)


def launches(fn):
    before = hecuda.kernel_launch_count()
    fn()
    return hecuda.kernel_launch_count() - before


def test_launches_do_not_grow_with_the_shard_count_and_past_32_shards_take_one_more_group():
    rng = np.random.default_rng(9)
    shapes = [RAGGED[i % len(RAGGED)] for i in range(33)]
    server = ragged_server(rng, shapes, np.uint64)
    requests = random_requests(rng, server, 3, 1)
    counts = {}
    for s in (1, 2, 5, 32, 33):
        sub = sp.SimplePirShardedServer(server.databases[:s], server.hints[:s], server.params[:s])
        reqs = [client[:s] for client in requests]
        counts[s] = launches(lambda: sub.computeResponses(reqs))
        got = sub.computeResponses(reqs)
        expect = per_shard_responses(sub, reqs)
        assert all(np.array_equal(got[c][i], expect[c][i]) for c in range(3) for i in range(s)), s
    assert counts[1] == counts[2] == counts[5] == counts[32] == 3  # split, grouped response, finish
    assert counts[33] == counts[32] + 2  # a second group: its split and its response


def test_grouped_response_at_the_accumulator_bound():
    """All-maximum operands over K = 2 x 32768 + 3 next to a small shard: every slice of the wide shard is full."""
    k = 2 * 32768 + 3
    prm_wide = sp.SimplePirParameters(enc(16, 61), 32, 1, 1, k)
    prm_small = sp.SimplePirParameters(enc(16, 61), 2 * 40, 1, 2, 70)
    wide = np.full((prm_wide.columnSize, k), (1 << 16) - 1, dtype=np.uint64)
    rng = np.random.default_rng(4)
    small = rng.integers(0, 1 << 16, size=(prm_small.columnSize, 70), dtype=np.uint64)
    server = sp.SimplePirShardedServer([sp.SimplePirDatabase.create(wide, prm_wide), sp.SimplePirDatabase.create(small, prm_small)],
                                       [np.zeros((prm_wide.columnSize, 16), np.uint64), np.zeros((prm_small.columnSize, 16), np.uint64)],
                                       [prm_wide, prm_small])
    requests = [[np.full((1, 1, k), np.iinfo(np.uint64).max, dtype=np.uint64),
                 rng.integers(0, 1 << 63, size=(1, 2, 70), dtype=np.uint64)] for _ in range(2)]
    got = server.computeResponses(requests)
    expect = ((1 << 16) - 1) * ((1 << 64) - 1) * k % (1 << 61)
    assert all(np.all(got[c][0] == np.uint64(expect)) for c in range(2))
    assert np.array_equal(got[1][1][0], osp.response(small, requests[1][1][0], 61))


def test_device_variant_matches_host_in_stream_order_and_graph_capture():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(5)
    server = ragged_server(rng, RAGGED, np.uint64)
    requests = random_requests(rng, server, 17, 2)
    flat_in = np.stack([np.concatenate([q.reshape(-1) for q in client]) for client in requests])
    host = server.computeResponses(flat_in, requests_per_shard=2)
    assert np.array_equal(host[3], np.concatenate([r.reshape(-1) for r in server.computeResponses(requests)[3]]))
    d_req = torch.from_numpy(flat_in.view(np.int64)).cuda()
    d_out = torch.zeros(host.shape, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        server.computeResponsesDevice(d_req.data_ptr(), 2, 17, d_out.data_ptr(), s.cuda_stream)
        got = d_out.clone()  # stream order: the clone runs after the response
    s.synchronize()
    assert np.array_equal(got.cpu().numpy().view(np.uint64), host)
    d_out.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        server.computeResponsesDevice(d_req.data_ptr(), 2, 17, d_out.data_ptr(), s.cuda_stream)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64), host)


def reference_flow(index):
    """simplePirFlow / simplePirFlowWithShardingOutOfBounds: 1000 rows x 50 B, chunk 15, 2 shards, N 1024, errorStdDev
    6.4, pt 14, ct 42, unchecked, through the all-shards client."""
    rng = np.random.default_rng(index)
    entries = rng.integers(0, 256, size=(1000, 50), dtype=np.uint8)
    server = sp.SimplePirShardedServer.process(entries, enc(14, 42, 1024, 6.4), 2, chunkSize=15, rng=rng)
    clients = [osp.Client(dict(N=1024, pt=14, ct=42, entries_per_column=p.entriesPerColumn,
                               chunks_per_entry=p.chunksPerEntry, database_columns=p.databaseColumns, entry_size=15),
                          h, p.seed, rng) for p, h in zip(server.params, server.hints)]
    mapped = [(e.originalIndex, e.size, [(c.shardIndex, c.index) for c in e.chunks]) for e in server.databaseMap.entries]
    client = ref.ClientForAllShards(mapped, 15, clients)
    queries = client.query(index)
    assert len({len(q) for q in queries}) == 1
    requests = [[np.stack([q[1][0] for q in qs]) for qs in queries]]  # one client, chunksPerShard requests per shard
    responses = server.computeResponses(requests)[0]
    return entries, client.decrypt([list(r) for r in responses], queries, index)


def test_reference_flow_with_sharding():
    entries, got = reference_flow(123)
    assert got == entries[123].tobytes()


def test_reference_flow_with_sharding_out_of_bounds():
    _, got = reference_flow(1100)
    assert got is None


def test_save_load_round_trip(tmp_path):
    rng = np.random.default_rng(8)
    server = sp.SimplePirShardedServer.process(variable_entries(rng, 100, 1, 60), enc(), 3, chunkSize=11,
                                               rng=np.random.default_rng(1))
    prefix = str(tmp_path / "db")
    server.save(prefix)
    assert (tmp_path / "db-2.bin").exists() and (tmp_path / "db-2.hint.bin").exists()
    again = sp.SimplePirShardedServer.load(prefix, server.params)
    for a, b in zip(again.databases, server.databases):
        assert np.array_equal(a.export(), b.export())
    assert all(np.array_equal(a, b) for a, b in zip(again.hints, server.hints))
    requests = random_requests(rng, server, 2, 1)
    got, expect = again.computeResponses(requests), server.computeResponses(requests)
    assert all(np.array_equal(a, b) for ca, cb in zip(got, expect) for a, b in zip(ca, cb))


def test_refusals_launch_nothing():
    lib = hecuda.load_library()
    rng = np.random.default_rng(2)
    entries = rng.integers(0, 256, size=(20, 30), dtype=np.uint8)  # 20 entries of 30 bytes, chunk 10: 3 chunks each
    offsets = np.arange(21, dtype=np.uint64) * np.uint64(30)
    good_locs = sp._chunk_locations(np.full(20, 30), 2, 10, np.random.default_rng(0))
    rows = np.bincount(good_locs[:, 0], minlength=2)
    params = [sp.SimplePirParameters.computingParams(enc(), int(r), 10, bytes(32)) for r in rows]
    seeds = np.zeros(64, dtype=np.uint8)
    hints = np.zeros(sum(p.columnSize for p in params) * 16, dtype=np.uint64)

    def process(locs=good_locs, prms=params, shard_count=2, chunk=10, values=entries, offs=offsets, count=20):
        cp = (sp._Params * len(prms))(*[p._c(64) if isinstance(p, sp.SimplePirParameters) else p for p in prms])
        out = (C.c_void_p * max(shard_count, 1))()
        rc = lib.hecuda_simple_pir_process_shards(None if values is None else values.ctypes.data, offs.ctypes.data,
                                                  count, chunk, shard_count, locs.ctypes.data, cp, seeds.ctypes.data,
                                                  hints.ctypes.data, out)
        for h in out:
            if h:
                lib.hecuda_simple_pir_database_destroy(h)
        return rc

    before = hecuda.kernel_launch_count()
    dup = good_locs.copy()
    dup[1] = dup[0]
    assert process(locs=dup) == -1  # not a permutation
    one = good_locs.copy()
    one[:, 0] = 0
    one[:, 1] = np.arange(60)
    assert process(locs=one) == -1  # shard 1 has no rows
    wrong_size = params[0]._c(64)
    wrong_size.entry_size = 11
    assert process(prms=[wrong_size, params[1]]) == -1
    wrong_count = params[0]._c(64)
    wrong_count.database_columns += 1
    assert process(prms=[wrong_count, params[1]]) == -1
    other_ct = params[1]._c(64)
    other_ct.ciphertext_modulus_bits = 41
    assert process(prms=[params[0], other_ct]) == -1
    assert process(values=None) == -1
    assert process(count=-1) == -1
    assert process(shard_count=0) == -1
    bad_offsets = offsets.copy()
    bad_offsets[3] = 0
    assert process(offs=bad_offsets) == -1
    assert hecuda.kernel_launch_count() == before
    assert process() == 0

    a = ragged_server(rng, RAGGED[:2], np.uint64)
    b = ragged_server(rng, RAGGED[:1], np.uint64, ct=41)
    c = ragged_server(rng, RAGGED[:1], np.uint32, ct=31)
    buf = np.zeros(1 << 16, dtype=np.uint64)
    before = hecuda.kernel_launch_count()

    def respond(dbs, shard_count=None, per_shard=1, req=buf, count=1, out=buf):
        handles = sp._handles(dbs)
        return lib.hecuda_simple_pir_compute_response_shards(handles, len(dbs) if shard_count is None else shard_count,
                                                             per_shard, None if req is None else req.ctypes.data, count,
                                                             None if out is None else out.ctypes.data)

    assert respond(a.databases + b.databases) == -1  # ct differs
    assert respond(a.databases + c.databases) == -1  # word_bits differ
    assert respond(a.databases, shard_count=0) == -1
    assert respond(a.databases, per_shard=0) == -1
    assert respond(a.databases, count=-1) == -1
    assert respond(a.databases, req=None) == -1
    assert respond(a.databases, out=None) == -1
    assert lib.hecuda_simple_pir_compute_response_shards(None, 1, 1, buf.ctypes.data, 1, buf.ctypes.data) == -1
    assert lib.hecuda_simple_pir_compute_response_shards((C.c_void_p * 1)(), 1, 1, buf.ctypes.data, 1,
                                                         buf.ctypes.data) == -1  # a null shard
    assert respond(a.databases, count=0) == 0  # nothing to answer
    assert hecuda.kernel_launch_count() == before
