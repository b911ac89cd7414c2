"""The two application workloads bench.py measures, at the benchmark's own shapes, bit-exact against the CPU oracle.

C4, MulPir computeResponse (tools/bench_pir.py): 2^20 entries of 64 B at N = 4096, t = 17 and the 27/28/28-bit PIR
moduli, so dimensions 437 x 75 over uint32 database rows, one query ciphertext expanded to 512, and 8 callers sharing
one server and one key through the captured response graph.  C5, PNNS mulTranspose (tools/bench_pnns.py): N = 8192,
t = 65537, a 100 000 x 512 matrix (13 result ciphertexts, baby and giant step 23) and a batch of 16 vectors with
modSwitchDownToSingle.

The fixtures draw the drivers' inputs from the drivers' seeds in the drivers' order, and the first test of each
workload proves it: the driver's own `run()` returns the same reply bit for bit.  So these tests check what the
benchmark computes, not a look-alike.  Every input comes from a fixed seed."""
import concurrent.futures
import ctypes
import gc
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir, pnns
from oracle import drbg_oracle as drbg
from oracle import oracle as orc
from oracle import pir_oracle as opir
from oracle import pnns_oracle as opn
from rlwe_shapes import read_device
from test_lazy_bounds_model import max_lazy_product_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _driver(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", f"{name}.py"))
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module


bench_pir = _driver("bench_pir")
bench_pnns = _driver("bench_pnns")

THREADS = 8     # bench_pir's concurrent callers
CALLS = 3       # calls per caller in the concurrency test
WORKERS = min(8, os.cpu_count() or 1)  # oracle thread pool: the C oracle releases the GIL


def _pool_map(fn, items):
    with concurrent.futures.ThreadPoolExecutor(WORKERS) as ex:
        return list(ex.map(fn, items))


def _free_device_bytes():
    """Free device memory once the driver has every block the library freed back: the library keeps the default
    pool's freed blocks for reuse (no release threshold), and the response graphs' allocations stay cached in the
    device's graph memory pool after the graphs are destroyed.  Both are caches, not leaks.  Also returns what the
    two pools still reserve, for the failure message."""
    import torch

    torch.cuda.synchronize()
    cuda = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cuda.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    assert cuda.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cuda.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0
    assert cuda.cuDeviceGraphMemTrim(dev) == 0
    pool_reserved, graph_reserved = ctypes.c_uint64(0), ctypes.c_uint64(0)
    cuda.cuMemPoolGetAttribute(pool, 5, ctypes.byref(pool_reserved))          # CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT
    cuda.cuDeviceGetGraphMemAttribute(dev, 2, ctypes.byref(graph_reserved))  # CU_GRAPH_MEM_ATTR_RESERVED_MEM_CURRENT
    held = f"default pool {pool_reserved.value >> 20} MiB, graph pool {graph_reserved.value >> 20} MiB, " \
           f"torch {torch.cuda.memory_reserved() >> 20} MiB reserved"
    return torch.cuda.mem_get_info()[0], held


@pytest.fixture(scope="module", autouse=True)
def no_device_leak():
    """Set up before and torn down after the workload fixtures: everything they and the drivers allocated is freed."""
    before, _ = _free_device_bytes()
    yield
    gc.collect()
    after, held = _free_device_bytes()
    leaked = before - after
    assert leaked < 64 << 20, f"the module leaves {leaked / 2**20:.1f} MiB of device memory allocated ({held})"


def widest_scan_sum(first, pts, cap):
    """The largest unreduced first-dimension sum sum_k first[k] pts[c, k] over columns c, polys and rows, as a Python
    integer.  first: (dim0, 2, L, N) Eval query; pts: (columns, dim0, L, N) Eval database.  Each half of the sum has
    at most cap = max_lazy_product_count(q, 64) products, so both halves are exact in uint64."""
    dim0 = first.shape[0]
    half = -(-dim0 // 2)
    assert half <= cap
    widest = 0
    for c in range(pts.shape[0]):
        for p in range(first.shape[1]):
            for r in range(first.shape[2]):
                a = (first[:half, p, r] * pts[c, :half, r]).sum(axis=0, dtype=np.uint64)
                b = (first[half:, p, r] * pts[c, half:, r]).sum(axis=0, dtype=np.uint64)
                floor_half = (a >> np.uint64(1)) + (b >> np.uint64(1)) + (((a & np.uint64(1)) + (b & np.uint64(1))) >> np.uint64(1))
                top = floor_half.max()
                widest = max(widest, max(int(a[i]) + int(b[i]) for i in np.flatnonzero(floor_half == top)))
    return widest


# ------------------------------------------------------------------------------------------------ C4: MulPir
class C4:
    """bench_pir.run's server, key and query (one GPU: RANK 0, WORLD_SIZE 1) and the oracle's replies."""

    ENTRIES, ENTRY_SIZE = 1 << 20, 64

    def __init__(self):
        n, t, moduli = 4096, 17, bench_pir.PIR_MODULI
        self.n, self.t = n, t
        self.g, self.o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
        L = self.L = self.g.L
        rng = np.random.default_rng(3)  # bench_pir.run's generator; the draws below follow its order
        config = (self.ENTRIES, self.ENTRY_SIZE, 2, 1, True, "hybridCompression", False)
        self.param = pir.MulPir.generateParameter(pir.IndexPirConfig(*config), self.g)
        self.oparam = opir.generate_parameter(opir.IndexPirConfig(*config), n, t)
        assert self.param.dimensions == self.oparam.dimensions == [437, 75]
        assert list(self.param.evaluationKeyConfig.galoisElements) == self.oparam.galois_elements
        chunk_count = -(-self.param.encodedEntrySize // pir.bytesPerPlaintext(self.g))
        assert chunk_count == 1
        count = chunk_count * int(np.prod(self.param.dimensions))
        rows = rng.integers(0, t, size=(count, n), dtype=np.uint64)
        self.db = pir.ProcessedDatabase(self.g, rows, None, evalFormat=False)
        self.server = pir.MulPirServer(self.param, self.g, [self.db])
        self.relin = bench_pir.uniform(rng, moduli, (L, 2), n)
        self.key = hecuda.EvaluationKey(self.g, self.relin)
        self.galois = {}
        for e in self.param.evaluationKeyConfig.galoisElements:
            self.galois[e] = bench_pir.uniform(rng, moduli, (L, 2), n)
            self.key.setGaloisKey(e, self.galois[e])
        query_cts = -(-self.param.expandedQueryCount // n)
        assert query_cts == 1 and self.param.expandedQueryCount == 512
        self.query = bench_pir.uniform(rng, moduli[:L], (query_cts, 2), n)
        self.packed = hecuda.Bfv.serialize(self.g, self.query[:, 0])
        self.seeds = rng.integers(0, 256, size=(query_cts, 32), dtype=np.uint8)
        # the oracle's database: the same Coeff rows through the oracle's NTT
        self.odb = opir._to_eval(self.o, rows)
        del rows
        # 8 callers, each with its own query
        self.thread_queries = bench_pir.uniform(np.random.default_rng(33), moduli[:L], (THREADS, query_cts, 2), n)
        self.wire_query = [drbg.expand_seeded_ciphertext(self.o, self.packed[i].tobytes(), self.seeds[i].tobytes())
                           for i in range(query_cts)]
        replies = _pool_map(self.oracle_reply, [list(self.query), self.wire_query] + [list(q) for q in self.thread_queries])
        self.expected, self.expected_wire, self.expected_threads = replies[0], replies[1], replies[2:]

    def oracle_reply(self, query):
        """The oracle's reply chunks, each (2, 1, N)."""
        return opir.compute_response(self.o, query, 1, self.galois, self.relin, [self.odb], self.oparam)[0]

    def close(self):
        self.key.close()
        self.db.close()
        self.g.close()


@pytest.fixture(scope="module")
def c4():
    s = C4()
    yield s
    s.close()


def assert_reply(got, expected, what):
    """got: (1, chunkCount, 2, 1, N) device reply; expected: the oracle's chunk list."""
    assert got.shape == (1, len(expected)) + expected[0].shape, what
    for chunk, ct in enumerate(expected):
        assert np.array_equal(got[0, chunk], ct), f"{what}, chunk {chunk}"


def test_c4_reply_is_the_benchmarks_and_matches_the_oracle(c4):
    got = c4.server.computeResponse(c4.query, c4.key)
    assert_reply(got, c4.expected, "C4 query")
    # the fixture draws what the driver draws: its timed reply is this reply, bit for bit
    ran = bench_pir.run(c4.ENTRIES, c4.ENTRY_SIZE, THREADS, per_thread=1, cpu=False, warmup=0)
    assert ran["database_plaintexts"] == c4.db.count
    assert np.array_equal(ran["reply"], got)


def test_c4_wire_reply_matches_the_oracle(c4):
    """PirWire.computeResponse as the driver times it: seeded serialized query in, skipLSBs-packed reply out."""
    replies, skips = pir.PirWire.computeResponse(c4.server, c4.packed, c4.seeds, c4.key)
    q0 = c4.o.q[:1]
    assert skips == opir.skip_lsbs_for_decryption(c4.n, q0[0], c4.t)
    assert replies.shape[:2] == (1, len(c4.expected_wire))
    for chunk, ct in enumerate(c4.expected_wire):
        want = opir.serialize_poly(c4.n, q0, ct[0], skips[0]) + opir.serialize_poly(c4.n, q0, ct[1], skips[1])
        assert replies[0, chunk].tobytes() == want, f"chunk {chunk}"


def test_c4_concurrent_callers_with_distinct_queries(c4):
    """8 callers on one server and one key, each with its own query, 3 calls each: every reply is its own query's."""
    import threading

    replies = [[None] * CALLS for _ in range(THREADS)]
    errors = []
    start = threading.Barrier(THREADS)

    def caller(i):
        try:
            start.wait()
            for k in range(CALLS):
                replies[i][k] = c4.server.computeResponse(c4.thread_queries[i], c4.key)
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=caller, args=(i,)) for i in range(THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for i in range(THREADS):
        for k in range(CALLS):
            assert_reply(replies[i][k], c4.expected_threads[i], f"caller {i}, call {k}")


def test_c4_scan_carries_its_sums_past_2_64(c4):
    """The uint32-row scan accumulates 64-bit sums and reduces every max_lazy_product_count(q, 64) = 256 terms;
    C4's first dimension has 437.  Uniform operands cannot show that the reduction carries the sum: a product
    averages q^2 / 4, so 437 of them sum to about 2^62.8.  Here the database holds Eval values in the top 1/64 of
    each modulus and the query is c0 = (q - 1) / 512 in its first 512 coefficients with c1 = 0, which the expansion
    turns into q - 1 in every Eval slot: the sums reach about 1.7 x 2^64.  The reply must still be the oracle's."""
    g, o, n, L = c4.g, c4.o, c4.n, c4.L
    dim0 = c4.param.dimensions[0]
    cap = max_lazy_product_count(max(o.q), 64)
    assert dim0 > cap
    rng = np.random.default_rng(41)
    count = c4.db.count
    rows = np.empty((count, L, n), dtype=np.uint64)
    for r, q in enumerate(o.q):
        rows[:, r, :] = rng.integers(q - (q >> 6), q, size=(count, n), dtype=np.uint64)
    query = np.zeros((1, 2, L, n), dtype=np.uint64)
    for r, q in enumerate(o.q):
        query[0, 0, r, :512] = (q - 1) * pow(512, -1, q) % q
    db = pir.ProcessedDatabase(g, rows, None, evalFormat=True)
    try:
        server = pir.MulPirServer(c4.param, g, [db])
        odb = opir.ProcessedDatabase(rows, np.ones(count, dtype=np.uint8))
        expanded = opir.expand(o, list(query), c4.oparam.expanded_query_count, c4.galois)
        first = np.stack([np.stack([orc.ntt_forward(n, o.q, ct[p]) for p in range(2)]) for ct in expanded[:dim0]])
        assert all(np.all(first[:, 0, r] == q - 1) for r, q in enumerate(o.q)) and not first[:, 1].any()
        widest = widest_scan_sum(first, rows.reshape(-1, dim0, L, n), cap)
        assert widest >= 1 << 64  # without its in-loop reductions the accumulator would wrap
        expected = opir.compute_response(o, list(query), 1, c4.galois, c4.relin, [odb], c4.oparam)[0]
        assert_reply(server.computeResponse(query, c4.key), expected, "C4 shape, sums past 2^64")
    finally:
        db.close()


# ------------------------------------------------------------------------------------------------ C5: PNNS
class C5:
    """bench_pnns.run's matrix, key and batch (one GPU) and the oracle's products of every vector."""

    ROWS, DIM, BATCH = 100000, 512, 16

    def __init__(self):
        n, t, moduli = 8192, 65537, bench_pnns.Q8192
        self.n = n
        self.g, self.o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
        L = self.L = self.g.L
        rng = np.random.default_rng(5)  # bench_pnns.run's generator; the draws below follow its order
        self.bsgs = pnns.BabyStepGiantStep.forVectorDimension(self.DIM)
        self.obsgs = opn.BabyStepGiantStep.for_dimension(self.DIM)
        assert (self.bsgs.vectorDimension, self.bsgs.babyStep, self.bsgs.giantStep) == \
            (self.obsgs.vector_dimension, self.obsgs.baby_step, self.obsgs.giant_step) == (512, 23, 23)
        self.results = -(-self.ROWS // n)
        assert self.results == 13
        count = self.bsgs.vectorDimension * self.results
        self.plain = rng.integers(0, t, size=(count, n), dtype=np.uint64)
        self.matrix = pnns.PlaintextMatrix(self.g, pnns.MatrixDimensions(self.ROWS, self.DIM), None, self.bsgs,
                                           plaintexts=self.plain)
        self.key = hecuda.EvaluationKey(self.g, None)
        self.galois = {}
        # the driver iterates this set literal: the same two ints in the same order give the same iteration order
        for e in {pnns.GaloisElement.rotatingColumns(-1, n), pnns.GaloisElement.rotatingColumns(-self.bsgs.babyStep, n)}:
            self.galois[e] = bench_pnns.uniform(rng, moduli, (L, 2), n)
            self.key.setGaloisKey(e, self.galois[e])
        assert sorted(self.galois) == sorted(opn.evaluation_key_elements(n, self.DIM))
        self.vec = bench_pnns.uniform(rng, moduli[:L], (self.BATCH, 2), n)
        self.eval_rows = opn.plaintexts_to_eval(self.o, self.plain, L)
        self.expected = _pool_map(self.oracle_product, range(self.BATCH))
        self.expected_single = [[opn.mod_switch_down_to_single(self.o, ct) for ct in e] for e in self.expected]

    def oracle_product(self, i):
        return opn.mul_transpose_vector(self.o, None, self.ROWS, self.obsgs, self.vec[i], self.galois,
                                        eval_rows=self.eval_rows)

    def close(self):
        self.matrix.close()
        self.key.close()
        self.g.close()


@pytest.fixture(scope="module")
def c5():
    s = C5()
    yield s
    s.close()


def test_c5_reply_is_the_benchmarks_and_matches_the_oracle(c5):
    got = c5.matrix.mulTranspose(c5.vec, c5.key, modSwitchDownToSingle=True)
    assert got.shape == (c5.BATCH, c5.results, 2, 1, c5.n)
    for i in range(c5.BATCH):
        for r in range(c5.results):
            assert np.array_equal(got[i, r], c5.expected_single[i][r]), f"vector {i}, result {r}"
    # the fixture draws what the driver draws: its timed batch reply is this reply, bit for bit
    ran = bench_pnns.run(c5.ROWS, c5.DIM, c5.BATCH, reps=1, cpu=False, warmup=0)
    assert ran["database_plaintexts"] == len(c5.plain)
    assert np.array_equal(ran["reply"], got)


def test_c5_batch_is_independent_of_its_vectors_positions(c5):
    """Every vector of the 16-batch against its own single-vector call, with and without modSwitchDownToSingle."""
    full = c5.matrix.mulTranspose(c5.vec, c5.key)
    assert full.shape == (c5.BATCH, c5.results, 2, c5.L, c5.n)
    for i in range(c5.BATCH):
        for r in range(c5.results):
            assert np.array_equal(full[i, r], c5.expected[i][r]), f"vector {i}, result {r}"
    single = c5.matrix.mulTranspose(c5.vec, c5.key, modSwitchDownToSingle=True)
    for i in range(c5.BATCH):
        assert np.array_equal(c5.matrix.mulTranspose(c5.vec[i:i + 1], c5.key)[0], full[i]), f"vector {i}"
        alone = c5.matrix.mulTranspose(c5.vec[i:i + 1], c5.key, modSwitchDownToSingle=True)[0]
        assert np.array_equal(alone, single[i]), f"vector {i}, modSwitchDownToSingle"


def test_c5_plaintext_rows_are_in_the_oracles_order(c5):
    """The `plaintexts=` constructor takes diagonal d = j + babyStep g of result ciphertext r from row
    resultCount d + r, as the oracle's mulTranspose reads it; the device keeps it at slot [r][g][j].  A transposed
    upload (row r vectorDimension + d) would put other rows in these slots."""
    b = c5.bsgs
    resident = read_device(*c5.matrix.deviceBuffer()).reshape(c5.results, b.giantStep, b.babyStep, c5.L, c5.n)
    present = c5.matrix.presentFlags().reshape(c5.results, b.giantStep, b.babyStep)
    diagonal = np.arange(b.babyStep)[None, :] + b.babyStep * np.arange(b.giantStep)[:, None]  # [g][j]
    used = diagonal < b.vectorDimension
    assert np.array_equal(present, np.broadcast_to(used, present.shape).astype(np.uint8))
    for r in range(c5.results):
        assert np.array_equal(resident[r][used], c5.eval_rows[c5.results * diagonal[used] + r]), f"result {r}"
