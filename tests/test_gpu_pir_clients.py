"""Many clients' MulPir queries in one call (hecuda_mulpir_compute_response_clients): every client has its own secret
key, relinearization key and Galois keys, and its reply must be bit-identical to the single-client call and to the
oracle, and decrypt to its database entry."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir
from oracle import oracle as orc
from oracle import pir_oracle as opir

TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)
PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:357-367)
GROUP = 16  # HECUDA_MULPIR_CLIENT_GROUP
TILE = 4    # clients per thread of the first-dimension scan (kScanClientTile)
ERR_INVALID_ARGUMENT, ERR_MISSING_KEY = -1, -5  # HECUDA_ERR_*

CONFIGS = [  # the configurations of test_gpu_pir.py
    dict(entry_size=1, dims=2, uneven=False, compression="noCompression"),
    dict(entry_size=8, dims=2, uneven=False, compression="noCompression"),
    dict(entry_size=24, dims=2, uneven=True, compression="noCompression"),
    dict(entry_size=24, dims=1, uneven=True, compression="noCompression"),
    dict(entry_size=24, dims=1, uneven=True, compression="hybridCompression"),
    dict(entry_size=24, dims=1, uneven=True, compression="maxCompression"),
    dict(entry_size=47, dims=2, uneven=True, compression="hybridCompression"),   # 3 chunks, two dimensions
]


class Setup:
    """One server (context, parameter, databases) and its oracle twin."""

    def __init__(self, g, o, entries, entry_size, dims, batch, uneven, compression, encoding=False, databases=1, seed=0):
        self.g, self.o = g, o
        rng = random.Random(seed)
        self.rng = rng
        self.param = pir.MulPir.generateParameter(
            pir.IndexPirConfig(entries, entry_size, dims, batch, uneven, compression, encoding), g)
        self.oparam = opir.generate_parameter(
            opir.IndexPirConfig(entries, entry_size, dims, batch, uneven, compression, encoding), o.n, o.t)
        assert self.param.dimensions == self.oparam.dimensions
        self.dbs = [[bytes(rng.randrange(256) for _ in range(rng.randint(1, entry_size) if encoding else entry_size))
                     for _ in range(entries)] for _ in range(databases)]
        self.server = pir.MulPirServer(self.param, g, [pir.MulPirServer.process(d, g, self.param) for d in self.dbs])
        self.odbs = [opir.process_database(o, self.oparam, d) for d in self.dbs]
        self.entries = entries

    def client(self, seed, indices_count=1, elements=None):
        o = self.o
        sk, relin = o.keygen(seed)
        key = hecuda.EvaluationKey(self.g, relin)
        okeys = {}
        for i, e in enumerate(self.param.evaluationKeyConfig.galoisElements if elements is None else elements):
            okeys[e] = o.galois_keygen(7000 + 31 * seed + i, sk, e)
            key.setGaloisKey(e, okeys[e])
        indices = [self.rng.randrange(self.entries) for _ in range(indices_count)]
        query = np.stack(opir.generate_query(o, self.oparam, indices, sk, 9000 + seed))
        return dict(sk=sk, relin=relin, key=key, okeys=okeys, indices=indices, query=query)

    def check(self, clients, indices_count=1, oracle_clients=None):
        """computeResponses == per-client computeResponse == oracle (for `oracle_clients`, default all), and decrypts."""
        got = self.server.computeResponses(np.stack([c["query"] for c in clients]), [c["key"] for c in clients],
                                           indicesCount=indices_count)
        chunks = self.server.chunkCount
        assert got.shape == (len(clients), indices_count, chunks, 2, 1, self.o.n)
        for j, c in enumerate(clients):
            single = self.server.computeResponse(c["query"], c["key"], indicesCount=indices_count)
            assert np.array_equal(got[j], single), f"client {j} differs from the single-client call"
            if oracle_clients is None or j in oracle_clients:
                expected = opir.compute_response(self.o, list(c["query"]), indices_count, c["okeys"], c["relin"], self.odbs,
                                                 self.oparam)
                for qi in range(indices_count):
                    for chunk in range(chunks):
                        assert np.array_equal(got[j, qi, chunk], expected[qi][chunk]), (j, qi, chunk)
            reply = [[got[j, qi, chunk] for chunk in range(chunks)] for qi in range(indices_count)]
            want = [self.dbs[qi if len(self.dbs) > 1 else 0][i] for qi, i in enumerate(c["indices"])]
            assert opir.decrypt_response(self.o, self.oparam, reply, c["indices"], c["sk"]) == want, f"client {j}"
        return got

    def close(self, clients):
        for c in clients:
            c["key"].close()


def contexts(n, bits, t):
    moduli = orc.generate_primes(bits, False, n)
    return hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)


@pytest.mark.parametrize("encoding", [False, True])
@pytest.mark.parametrize("cfg", CONFIGS)
def test_clients_match_single_client_and_oracle(cfg, encoding):
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 100, cfg["entry_size"], cfg["dims"], 1, cfg["uneven"], cfg["compression"], encoding,
              seed=cfg["entry_size"] * 3 + cfg["dims"] + 17 * encoding)
    clients = [s.client(40 + c) for c in range(3)]
    s.check(clients)
    s.close(clients)
    g.close()


@pytest.mark.parametrize("count", [1, 2, 3, TILE, TILE + 1, GROUP, GROUP + 1])
def test_client_counts(count):
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 100, 47, 2, 1, True, "hybridCompression", seed=count)
    clients = [s.client(100 + c) for c in range(count)]
    s.check(clients)
    s.close(clients)
    g.close()


@pytest.mark.parametrize("databases", [1, 2])
def test_two_indices_per_client(databases):
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 40, 4, 2, 2, False, "noCompression", databases=databases, seed=5 + databases)
    clients = [s.client(200 + c, indices_count=2) for c in range(TILE + 1)]
    s.check(clients, indices_count=2)
    s.close(clients)
    g.close()


@pytest.mark.parametrize("n,bits,t,entries,entry_size,compression,count", [
    (4096, [27, 28, 28], 17, 30000, 1, "hybridCompression", TILE + 1),   # uint32 database rows
    (8192, [55, 55, 55, 55], 65537, 5000, 100, "maxCompression", 2),    # uint64 database rows
])
def test_production_sizes(n, bits, t, entries, entry_size, compression, count):
    g, o = contexts(n, bits, t)
    s = Setup(g, o, entries, entry_size, 2, 1, True, compression, seed=entries)
    clients = [s.client(300 + c) for c in range(count)]
    s.check(clients, oracle_clients={0, count - 1})
    s.close(clients)
    g.close()


def test_32_bit_context():
    n, t = 4096, 17
    g, o = hecuda.Context(n, PIR_MODULI, t, scalar=np.uint32), orc.Context(n, PIR_MODULI, t, word_bits=32)
    s = Setup(g, o, 20000, 1, 2, 1, True, "hybridCompression", seed=32)
    clients = [s.client(400 + c) for c in range(3)]
    s.check(clients, oracle_clients={1})
    s.close(clients)
    g.close()


def _raw_call(s, keys, queries, indices_count=1, databases=None):
    """hecuda_mulpir_compute_response_clients with raw handles (None = a null evk)."""
    dbs = s.server.databases if databases is None else databases
    q = np.ascontiguousarray(queries, dtype=np.uint64)
    count = len(keys)
    out = np.empty((max(count, 1), indices_count, s.server.chunkCount, 2, 1, s.o.n), dtype=np.uint64)
    handles = (C.c_void_p * len(dbs))(*[d._h for d in dbs])
    key_handles = (C.c_void_p * max(count, 1))(*[k._h if k is not None else None for k in keys])
    dims = (C.c_int32 * len(s.param.dimensions))(*s.param.dimensions)
    qct = q.shape[1] if q.ndim == 5 else 1
    hecuda._check(hecuda.load_library().hecuda_mulpir_compute_response_clients(
        s.g._h, key_handles, count, handles, len(dbs), dims, len(dims), s.server.chunkCount,
        q.ctypes.data_as(C.c_void_p), qct, indices_count, out.ctypes.data_as(C.c_void_p)))
    return out


def test_errors():
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 40, 4, 2, 1, False, "noCompression", seed=77)
    clients = [s.client(500 + c) for c in range(3)]
    queries = np.stack([c["query"] for c in clients])
    keys = [c["key"] for c in clients]
    with pytest.raises(hecuda.HeError) as err:  # client_count 0
        _raw_call(s, [], queries[:1])
    assert err.value.code == ERR_INVALID_ARGUMENT
    with pytest.raises(hecuda.HeError) as err:  # a null evk
        _raw_call(s, [keys[0], None, keys[2]], queries)
    assert err.value.code == ERR_MISSING_KEY and "client 1" in str(err.value)
    g2, _ = contexts(16, TEST_MODULI_BITS, 1153)  # an evk of another context
    foreign = hecuda.EvaluationKey(g2, clients[0]["relin"])
    with pytest.raises(hecuda.HeError) as err:
        s.server.computeResponses(queries, [keys[0], keys[1], foreign])
    assert err.value.code == ERR_INVALID_ARGUMENT and "client 2" in str(err.value)
    foreign.close()
    g2.close()
    elements = s.param.evaluationKeyConfig.galoisElements
    partial = s.client(600, elements=[e for e in elements if e != min(elements)])  # misses the last level's key
    with pytest.raises(hecuda.HeError) as err:
        s.server.computeResponses(np.stack([queries[0], partial["query"]]), [keys[0], partial["key"]])
    assert err.value.code == ERR_MISSING_KEY and "client 1" in str(err.value) and "missingGaloisKey" in str(err.value)
    bare = hecuda.EvaluationKey(g, None)  # one client misses its relinearization key
    for e, k in clients[2]["okeys"].items():
        bare.setGaloisKey(e, k)
    with pytest.raises(hecuda.HeError) as err:
        s.server.computeResponses(queries, [keys[0], keys[1], bare])
    assert err.value.code == ERR_MISSING_KEY and "client 2" in str(err.value)
    assert "missingRelinearizationKey" in str(err.value)
    bare.close()
    # Galois element sets that resolve differently: maxCompression keys (x -> x^9 applied twice at the first level)
    # against noCompression keys (x -> x^17 once)
    compressed = pir.MulPir.evaluationKeyConfig(s.param.expandedQueryCount, o.n, "maxCompression").galoisElements
    assert sorted(compressed) != sorted(elements)
    low = s.client(700, elements=compressed)
    single = s.server.computeResponse(low["query"], low["key"])  # the single-client call serves it
    reply = [[single[0, c] for c in range(s.server.chunkCount)]]
    assert opir.decrypt_response(o, s.oparam, reply, low["indices"], low["sk"]) == [s.dbs[0][low["indices"][0]]]
    with pytest.raises(hecuda.HeError) as err:
        s.server.computeResponses(np.stack([queries[0], low["query"]]), [keys[0], low["key"]])
    assert err.value.code == ERR_INVALID_ARGUMENT and "client 1" in str(err.value)
    with pytest.raises(hecuda.HeError) as err:  # PirError.invalidBatchSize: 2 databases, 3 indices
        _raw_call(s, keys[:1], np.zeros((1, queries.shape[1], 2, o.L, o.n), dtype=np.uint64), indices_count=3,
                  databases=s.server.databases * 2)
    assert "invalidBatchSize" in str(err.value)
    s.close(clients + [partial, low])
    g.close()


def test_launch_count_does_not_depend_on_the_group_size():
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 100, 47, 2, 1, True, "hybridCompression", seed=3)
    clients = [s.client(800 + c) for c in range(GROUP)]
    queries = np.stack([c["query"] for c in clients])
    keys = [c["key"] for c in clients]

    def launches(count):
        before = hecuda.kernel_launch_count()
        s.server.computeResponses(queries[:count], keys[:count])
        return hecuda.kernel_launch_count() - before

    launches(2)  # the first call uploads the expansion plan
    assert launches(2) == launches(GROUP) == launches(TILE + 1)
    s.close(clients)
    g.close()


def test_device_variant_and_concurrent_callers():
    import torch

    g, o = contexts(64, [55, 55, 55], 65537)
    s = Setup(g, o, 200, 24, 2, 1, True, "hybridCompression", seed=9)
    clients = [s.client(900 + c) for c in range(TILE + 2)]
    queries = np.stack([c["query"] for c in clients])
    keys = [c["key"] for c in clients]
    want = s.check(clients, oracle_clients={0})
    # _device on a caller's stream
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        d_q = torch.from_numpy(queries.view(np.int64)).cuda()
        d_out = torch.empty((len(clients),) + want.shape[1:], dtype=torch.int64, device="cuda")
    stream.synchronize()
    dbs = s.server.databases
    handles = (C.c_void_p * len(dbs))(*[d._h for d in dbs])
    key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
    dims = (C.c_int32 * len(s.param.dimensions))(*s.param.dimensions)
    hecuda._check(hecuda.load_library().hecuda_mulpir_compute_response_clients_device(
        g._h, key_handles, len(keys), handles, len(dbs), dims, len(dims), s.server.chunkCount, d_q.data_ptr(),
        queries.shape[1], 1, d_out.data_ptr(), stream.cuda_stream))
    stream.synchronize()
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64), want)
    # two host threads, each with its own clients
    halves = [list(range(0, 3)), list(range(3, len(clients)))]
    results, errors = {}, []

    def worker(tid):
        try:
            for _ in range(2):
                idx = halves[tid]
                results[tid] = s.server.computeResponses(queries[idx], [keys[i] for i in idx])
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for tid, idx in enumerate(halves):
        assert np.array_equal(results[tid], want[idx])
    s.close(clients)
    g.close()


@pytest.mark.parametrize("count,faulty", [(GROUP + 1, GROUP), (GROUP + 2, GROUP + 1)])
def test_errors_in_a_later_group_name_the_client_and_enqueue_nothing(count, faulty):
    """A key problem of a client in the second group (alone there, or beside another client) is reported with its index
    in the call, before any group runs: the device variant leaves the output buffer untouched."""
    import re

    import torch

    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 40, 4, 2, 1, False, "noCompression", seed=faulty)
    clients = [s.client(1100 + c) for c in range(count)]
    elements = s.param.evaluationKeyConfig.galoisElements
    compressed = pir.MulPir.evaluationKeyConfig(s.param.expandedQueryCount, o.n, "maxCompression").galoisElements
    missing = s.client(1200, elements=[e for e in elements if e != min(elements)])   # misses the last level's key
    different = s.client(1300, elements=compressed)                                  # resolves to other elements
    dbs = s.server.databases
    handles = (C.c_void_p * len(dbs))(*[d._h for d in dbs])
    dims = (C.c_int32 * len(s.param.dimensions))(*s.param.dimensions)
    stream = torch.cuda.Stream()
    for bad, code in ((missing, ERR_MISSING_KEY), (different, ERR_INVALID_ARGUMENT)):
        batch = clients[:faulty] + [bad] + clients[faulty + 1:]
        queries = np.stack([c["query"] for c in batch])
        with pytest.raises(hecuda.HeError) as err:
            s.server.computeResponses(queries, [c["key"] for c in batch])
        assert err.value.code == code and re.search(rf"\bclient {faulty}\b", str(err.value)), str(err.value)
        with torch.cuda.stream(stream):
            d_q = torch.from_numpy(queries.view(np.int64)).cuda()
            d_out = torch.full((count, 1, s.server.chunkCount, 2, 1, o.n), 7, dtype=torch.int64, device="cuda")
        stream.synchronize()
        key_handles = (C.c_void_p * count)(*[c["key"]._h for c in batch])
        rc = hecuda.load_library().hecuda_mulpir_compute_response_clients_device(
            g._h, key_handles, count, handles, len(dbs), dims, len(dims), s.server.chunkCount, d_q.data_ptr(),
            queries.shape[1], 1, d_out.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        assert rc == code
        assert bool((d_out == 7).all()), "a failed call wrote part of the replies"
    s.close(clients + [missing, different])
    g.close()
