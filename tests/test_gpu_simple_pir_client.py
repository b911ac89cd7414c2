"""SimplePIR's device client (hecuda.simple_pir.DefaultQueryGenerator / SimplePirClient over
csrc/simple_pir_client.cu): seeded precompute bit-exact against tests/simple_pir_client_ref.py over both scalars,
several N, ct, errorStdDev, chunksPerEntry, aPolyCount and counts; the results product where the reference's
double-width sum wraps; decryption on crafted responses at the rounding edges; round trips with the device server,
sharded flows, stream order and graph capture, launch counts for absent indices, validation, and refusals."""
import ctypes as C

import numpy as np
import pytest

import hecuda
import simple_pir_client_ref as ref
from hecuda import simple_pir as sp
from oracle import simple_pir_oracle as osp
from oracle.pir_oracle import coefficients_to_bytes

pytestmark = pytest.mark.gpu


def enc(pt, ct, n, std=3.2):
    return sp.SimplePirEncryptionParams(pt, ct, n, std, "unchecked")


def seeds(rng, count):
    return [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(count)]


# (scalar, N, pt, ct, errorStdDev, entry bytes, entriesPerColumn, chunksPerEntry, databaseColumns, count, indexed)
SHAPES = [
    (np.uint32, 8, 4, 9, 3.2, 3, 5, 1, 7, 1, False),
    (np.uint32, 16, 7, 28, 6.4, 20, 1, 3, 37, 7, True),     # cpe > 1, aPolyCount 3 with K not a multiple of N
    (np.uint32, 16, 9, 31, 3.2, 40, 2, 1, 40, 33, True),    # M = 72: not a multiple of the 128-row CTA
    (np.uint64, 16, 14, 42, 6.4, 60, 1, 2, 50, 7, False),
    (np.uint64, 16, 16, 61, 3.2, 30, 3, 1, 20, 33, True),   # 8 hint planes
    (np.uint32, 1024, 9, 28, 3.2, 12, 1, 1, 1500, 1, True),
    (np.uint64, 2048, 14, 42, 6.4, 256, 1, 2, 2100, 7, True),
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{np.dtype(s[0]).name}-N{s[1]}-ct{s[3]}-q{s[9]}")
def test_precompute_is_bit_exact(shape):
    scalar, n, pt, ct, std, size, epc, cpe, k, count, indexed = shape
    rng = np.random.default_rng(n + ct + count)
    prm = sp.SimplePirParameters(enc(pt, ct, n, std), size, epc, cpe, k, seeds(rng, 1)[0])
    p = osp.ntt_friendly_mod(ct, n)
    hint = rng.integers(0, p, size=(prm.columnSize, n), dtype=np.uint64).astype(scalar)
    gen = sp.DefaultQueryGenerator(prm, hint, scalar)
    ss, es = seeds(rng, count), seeds(rng, count)
    indices = rng.integers(0, (k * epc - cpe) // cpe + 1, size=count) if indexed else None
    q, r = gen.precompute(count, indices, ss, es)
    d = dict(N=n, pt=pt, ct=ct, entries_per_column=epc, chunks_per_entry=cpe, database_columns=k)
    bits = np.dtype(scalar).itemsize * 8
    for i in sorted({0, count - 1, count // 2}):  # the Python AES is slow: three of the queries
        eq, er, _ = ref.precompute(d, hint, prm.seed, ss[i], es[i], None if indices is None else int(indices[i]), bits, std)
        assert np.array_equal(q[i].astype(np.uint64), eq), i
        assert np.array_equal(r[i].astype(np.uint64), er), i


@pytest.mark.parametrize("scalar,ct,wraps", [(np.uint32, 28, True), (np.uint64, 42, False)])
def test_results_at_the_largest_hint(scalar, ct, wraps):
    """Every hint word p - 1: at UInt32 ct 28 N 1024 the reference's double-width sum wraps (the device must wrap the
    same way); at UInt64 ct 42 it does not."""
    n = 1024 if scalar == np.uint32 else 2048
    rng = np.random.default_rng(ct)
    p = osp.ntt_friendly_mod(ct, n)
    prm = sp.SimplePirParameters(enc(8, ct, n), 40, 1, 1, 64, seeds(rng, 1)[0])
    hint = np.full((prm.columnSize, n), p - 1, dtype=scalar)
    gen = sp.DefaultQueryGenerator(prm, hint, scalar)
    ss = seeds(rng, 2)
    _, r = gen.precompute(2, None, ss, seeds(rng, 2))
    bits = np.dtype(scalar).itemsize * 8
    for i in range(2):
        s = ref.secrets_from_seed(ss[i], 1, n)
        wrapped, exact = ref.results(s, hint, p, bits), ref.results(s, hint, p, bits, exact=True)
        assert np.array_equal(r[i].astype(np.uint64), wrapped)
        assert (not np.array_equal(wrapped, exact)) == wraps


@pytest.mark.parametrize("scalar,pt,ct,epc,cpe", [(np.uint32, 9, 28, 3, 1), (np.uint64, 14, 42, 1, 3),
                                                  (np.uint64, 1, 8, 2, 1)])
def test_decrypt_is_bit_exact_at_the_rounding_edges(scalar, pt, ct, epc, cpe):
    rng = np.random.default_rng(pt)
    size = 25
    prm = sp.SimplePirParameters(enc(pt, ct, 16), size, epc, cpe, 9, bytes(32))
    p = osp.ntt_friendly_mod(ct, 16)
    client = sp.SimplePirClient(sp.DefaultQueryGenerator(prm, np.zeros((prm.columnSize, 16), scalar), scalar))
    delta, mask = 1 << (ct - pt), (1 << ct) - 1
    count = 6
    results = rng.integers(0, p, size=(count, cpe, prm.columnSize), dtype=np.uint64)
    plain = rng.integers(0, 1 << pt, size=(count, cpe, prm.columnSize), dtype=np.uint64)
    # r - s = m delta + offset with offset delta/2 - 1 (rounds down), -delta/2 (rounds up to m), and a mask wrap
    offsets = np.array([delta // 2 - 1, -(delta // 2), -1, 0, delta // 2 - 1, -(delta // 2)], dtype=object)
    resp = ((plain.astype(object) * delta + offsets[:, None, None] + results.astype(object)) & mask).astype(np.uint64)
    indices = rng.integers(0, 3, size=count)
    got = client.decryptMany(resp.astype(scalar), results.astype(scalar), indices)
    chunk = prm.chunkSize
    for qi in range(count):
        coeffs = []
        for i in range(cpe):
            start = ((indices[qi] * cpe + i) % epc) * chunk
            for c in range(start, start + chunk):
                v = (int(resp[qi, i, c]) - int(results[qi, i, c]) + (delta >> 1)) & mask
                coeffs.append(v >> (ct - pt))
        assert got[qi].tobytes() == coefficients_to_bytes(np.array(coeffs, dtype=np.uint64), pt)[:size], qi


def round_trip_setup(scalar, pt, ct, n, std, entries):
    results = sp.SimplePirServer.process(entries, enc(pt, ct, n, std), scalar=scalar)
    server = sp.SimplePirServer(results.database, results.hint, results.params, scalar)
    return server, sp.SimplePirClient(sp.DefaultQueryGenerator(results.params, results.hint, scalar))


@pytest.mark.parametrize("scalar,pt,ct", [(np.uint32, 7, 28), (np.uint64, 14, 42)])
def test_encrypt_decrypt_round_trip(scalar, pt, ct):
    """runEncryptDecryptRoundTripTest: query(at:), computeResponse, decrypt, for several entries; then the batched
    forms."""
    rng = np.random.default_rng(ct)
    entries = rng.integers(0, 256, size=(300, 24), dtype=np.uint8)
    server, client = round_trip_setup(scalar, pt, ct, 1024, 3.2, entries)
    for index in (0, 7, 299):
        q = client.query(index)
        assert client.decrypt(server.computeResponse(q.queries), q.prepareResponse(), index) == entries[index].tobytes()
    idx = [5, 5, 123, 299, 0]
    qs = client.queries(idx)
    responses = server.computeResponses(np.stack([q.queries for q in qs]))
    got = client.decryptMany(responses, np.stack([q.resultsWithoutResponse for q in qs]), idx)
    assert all(got[i].tobytes() == entries[ix].tobytes() for i, ix in enumerate(idx))


def test_device_calls_in_stream_order_and_one_graph():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    entries = rng.integers(0, 256, size=(200, 40), dtype=np.uint8)
    server, client = round_trip_setup(np.uint64, 14, 42, 1024, 6.4, entries)
    p = server.params
    count, idx = 5, np.array([1, 199, 50, 50, 0], dtype=np.int64)
    ss, es = seeds(rng, count), seeds(rng, count)
    hq, hr = client.queryGenerator.precompute(count, idx, ss, es)
    d_ss = torch.from_numpy(np.frombuffer(b"".join(ss), dtype=np.uint8).copy()).cuda()
    d_es = torch.from_numpy(np.frombuffer(b"".join(es), dtype=np.uint8).copy()).cuda()
    d_idx = torch.from_numpy(idx).cuda()
    d_q = torch.zeros((count, p.chunksPerEntry, p.databaseColumns), dtype=torch.int64, device="cuda")
    d_r = torch.zeros((count, p.chunksPerEntry, p.columnSize), dtype=torch.int64, device="cuda")
    d_resp = torch.zeros_like(d_r)
    d_out = torch.zeros((count, p.entrySizeInBytes), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()

    def pipeline():
        client.precomputeDevice(d_ss.data_ptr(), d_es.data_ptr(), d_idx.data_ptr(), count, d_q.data_ptr(), d_r.data_ptr(),
                                s.cuda_stream)
        server.computeResponsesDevice(d_q.data_ptr(), count, d_resp.data_ptr(), s.cuda_stream)
        client.decryptDevice(d_resp.data_ptr(), d_r.data_ptr(), d_idx.data_ptr(), count, d_out.data_ptr(), s.cuda_stream)

    with torch.cuda.stream(s):
        pipeline()
        q_copy, out_copy = d_q.clone(), d_out.clone()  # stream order: the clones run after the calls
    s.synchronize()
    assert np.array_equal(q_copy.cpu().numpy().view(np.uint64), hq)
    assert np.array_equal(d_r.cpu().numpy().view(np.uint64), hr)
    assert all(out_copy.cpu().numpy()[i].tobytes() == entries[ix].tobytes() for i, ix in enumerate(idx))
    for t in (d_q, d_r, d_resp, d_out):
        t.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        pipeline()
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(d_q.cpu().numpy().view(np.uint64), hq)
    assert all(d_out.cpu().numpy()[i].tobytes() == entries[ix].tobytes() for i, ix in enumerate(idx))


def sharded(rng, scalar=np.uint64):
    """simplePirFlowWithSharding: 1000 rows x 50 B, chunk 15, 2 shards, N 1024, errorStdDev 6.4, pt 14, ct 42."""
    entries = rng.integers(0, 256, size=(1000, 50), dtype=np.uint8)
    server = sp.SimplePirShardedServer.process(entries, enc(14, 42, 1024, 6.4), 2, chunkSize=15, rng=rng, scalar=scalar)
    clients = [sp.SimplePirClient(sp.DefaultQueryGenerator(p, h, scalar)) for p, h in zip(server.params, server.hints)]
    return entries, server, sp.SimplePirClientForAllShards(server.databaseMap, clients)


def shard_flow(server, client, index):
    queries = client.query(index)
    requests = [[np.stack([q.queries for q in qs]) for qs in queries]]
    responses = server.computeResponses(requests)[0]
    return client.decrypt([list(r) for r in responses], index, queries)


def test_sharded_flow_and_out_of_bounds():
    rng = np.random.default_rng(11)
    entries, server, client = sharded(rng)
    assert shard_flow(server, client, 123) == entries[123].tobytes()
    assert shard_flow(server, client, 1100) is None


def test_absent_index_launches_what_a_present_one_does():
    rng = np.random.default_rng(12)
    _, server, client = sharded(rng)
    counts = []
    for index in (5, 1100):
        before = hecuda.kernel_launch_count()
        shard_flow(server, client, index)
        counts.append(hecuda.kernel_launch_count() - before)
    assert counts[0] == counts[1] > 0


def test_batched_sharded_queries_feed_the_grouped_response():
    rng = np.random.default_rng(13)
    entries, server, client = sharded(rng)
    idx = [0, 999, 1100, 500]
    flat, queries = client.queriesMany(idx)
    per = client.queriesPerShard
    out = server.computeResponses(flat, requests_per_shard=per)
    bounds = np.concatenate([[0], np.cumsum(server._words(per)[1])])
    for c, index in enumerate(idx):
        responses = [out[c, bounds[s]:bounds[s + 1]].reshape(per, p.chunksPerEntry, p.columnSize)
                     for s, p in enumerate(server.params)]
        got = client.decrypt(responses, index, queries[c])
        assert got == (entries[index].tobytes() if index < 1000 else None)


def test_validate_passes_and_catches_a_changed_value():
    rng = np.random.default_rng(14)
    entries = rng.integers(0, 256, size=(400, 100), dtype=np.uint8)
    server = sp.SimplePirShardedServer.process(entries, enc(14, 42, 1024, 6.4), 5, rng=rng)
    index = 77
    times, value = server.validate((index, entries[index].tobytes()), trials=2)
    assert value == entries[index].tobytes() and len(times) == 2
    assert {c.shardIndex for c in server.databaseMap.entries[index].chunks} == set(range(5))  # spans every shard
    # change one DB' value inside the tested entry's first chunk
    loc = server.databaseMap.entries[index].chunks[0]
    prm = server.params[loc.shardIndex]
    db = server.databases[loc.shardIndex].export()
    row = (loc.index * prm.chunksPerEntry) % prm.entriesPerColumn * prm.chunkSize
    col = (loc.index * prm.chunksPerEntry) // prm.entriesPerColumn
    db[row, col] ^= 1
    bad = sp.SimplePirShardedServer(
        [sp.SimplePirDatabase.create(db, prm) if s == loc.shardIndex else d for s, d in enumerate(server.databases)],
        server.hints, server.params, databaseMap=server.databaseMap)
    with pytest.raises(sp.PirError, match=f"Verification failed for index {index}"):
        bad.validate((index, entries[index].tobytes()))
    single = sp.SimplePirServer.process(entries, enc(14, 42, 1024, 6.4))
    one = sp.SimplePirServer(single.database, single.hint, single.params)
    assert one.validate((3, entries[3].tobytes()))[1] == entries[3].tobytes()


def test_refusals_launch_nothing():
    lib = hecuda.load_library()
    prm = sp.SimplePirParameters(enc(14, 42, 16, 6.4), 30, 1, 1, 20, bytes(32))
    p = osp.ntt_friendly_mod(42, 16)
    hint = np.zeros((prm.columnSize, 16), np.uint64)
    gen = sp.DefaultQueryGenerator(prm, hint)
    buf = np.zeros(1 << 16, dtype=np.uint64)
    seed = np.zeros(64, dtype=np.uint8)
    before = hecuda.kernel_launch_count()
    bad = hint.copy()
    bad[2, 3] = p
    out = C.c_void_p()
    cp = prm._c(64)
    assert lib.hecuda_simple_pir_client_create(bad.ctypes.data, C.byref(cp), seed.ctypes.data, C.byref(out)) == -1
    assert lib.hecuda_simple_pir_client_create(None, C.byref(cp), seed.ctypes.data, C.byref(out)) == -1
    cp.ciphertext_modulus_bits = 14  # ct <= pt
    assert lib.hecuda_simple_pir_client_create(hint.ctypes.data, C.byref(cp), seed.ctypes.data, C.byref(out)) == -1

    def pre(count=1, idx=None, ss=seed, q=buf):
        i = None if idx is None else np.array(idx, dtype=np.int64)
        return lib.hecuda_simple_pir_client_precompute(gen._h, None if ss is None else ss.ctypes.data, seed.ctypes.data,
                                                       None if i is None else i.ctypes.data, count,
                                                       None if q is None else q.ctypes.data, buf.ctypes.data)

    assert pre(count=-1) == -1
    assert pre(ss=None) == -1
    assert pre(q=None) == -1
    assert pre(idx=[-1]) == -1
    assert pre(idx=[20]) == -1  # column 20 reaches K = 20
    assert pre(count=1 << 40) == -1
    assert pre(count=0) == 0
    idx = np.array([-1], dtype=np.int64)
    assert lib.hecuda_simple_pir_client_decrypt(gen._h, buf.ctypes.data, buf.ctypes.data, idx.ctypes.data, 1,
                                                buf.ctypes.data) == -1
    assert lib.hecuda_simple_pir_client_decrypt(gen._h, buf.ctypes.data, buf.ctypes.data, None, 1, buf.ctypes.data) == -1
    assert lib.hecuda_simple_pir_client_decrypt(None, buf.ctypes.data, buf.ctypes.data, idx.ctypes.data, 1,
                                                buf.ctypes.data) == -1
    assert hecuda.kernel_launch_count() == before
    assert pre(idx=[19]) == 0
