"""Many PNNS clients in one call (hecuda_pnns_compute_response_clients and its wire form): every client has its own
secret key and Galois keys; its replies must be bit-identical to the single-client mulTransposeMatrix +
modSwitchDownToSingle, to the oracle, and decrypt to M q mod t."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import evk_wire_ref as ref
import hecuda
from hecuda import pnns
from oracle import oracle as orc
from oracle import pir_oracle as opir
from oracle import pnns_oracle as opn
from test_gpu_evk_wire import seeded_keys

GROUP = 16  # HECUDA_PNNS_CLIENT_GROUP
ERR_INVALID_ARGUMENT, ERR_MISSING_KEY = -1, -5  # HECUDA_ERR_*
TEST_BITS = (55, 52, 62, 58)  # TestUtils.testCoefficientModuli for UInt64


class Server:
    """One context and plaintext matrix, their oracle twins, and the query shape every client uses."""

    def __init__(self, n, t, bits, rows, cols, queries, seed=0, moduli=None):
        moduli = moduli or orc.generate_primes(list(bits), False, n)
        self.g, self.o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
        self.n, self.t, self.rows, self.cols, self.queries = n, t, rows, cols, queries
        self.rng = random.Random(seed)
        self.values = [[self.rng.randrange(t) for _ in range(cols)] for _ in range(rows)]
        self.flat = [v for row in self.values for v in row]
        self.matrix = pnns.PlaintextMatrix(self.g, pnns.MatrixDimensions(rows, cols), self.flat)
        self.bsgs = opn.BabyStepGiantStep.for_dimension(cols)
        self.dims = pnns.MatrixDimensions(queries, cols)
        self.elements = opn.matrix_evaluation_key_elements(n, rows, cols, queries)
        self._oplain = None

    @property
    def oplain(self):
        if self._oplain is None:
            self._oplain = opn.diagonal_plaintexts(self.o, self.rows, self.cols, self.bsgs, self.flat)
        return self._oplain

    def query(self, seed, sk):
        rng = random.Random(seed)
        query = [[rng.randrange(self.t) for _ in range(self.cols)] for _ in range(self.queries)]
        plain = opn.dense_row_plaintexts(self.o, self.queries, self.cols, [v for row in query for v in row])
        return query, np.stack([self.o.encrypt(5000 + 37 * seed + i, sk, p) for i, p in enumerate(plain)])

    def client(self, seed, elements=None):
        o = self.o
        sk, _ = o.keygen(seed, relin=False)
        key, okeys = hecuda.EvaluationKey(self.g, None), {}
        for i, e in enumerate(self.elements if elements is None else elements):
            okeys[e] = o.galois_keygen(100 * seed + i, sk, e)
            key.setGaloisKey(e, okeys[e])
        query, cts = self.query(seed, sk)
        return dict(sk=sk, key=key, okeys=okeys, query=query, cts=cts)

    def oracle(self, c):
        """opn.mul_transpose_matrix + opn.mod_switch_down_to_single of client c."""
        out = opn.mul_transpose_matrix(self.o, self.oplain, self.rows, self.cols, self.bsgs, list(c["cts"]), self.queries,
                                       c["okeys"])
        return [opn.mod_switch_down_to_single(self.o, ct) for ct in out]

    def assert_decrypts(self, c, replies, who):
        decoded = [opn.decode_simd(self.o, self.o.decrypt(c["sk"], ct)).tolist() for ct in replies]
        want = [sum(a * b for a, b in zip(self.values[r], c["query"][q])) % self.t
                for r in range(self.rows) for q in range(self.queries)]
        assert opn.unpack_dense_column(self.o, decoded, self.rows, self.queries) == want, who

    def check(self, clients, oracle_clients=None):
        """computeResponses == per-client mulTransposeMatrix(modSwitchDownToSingle) == oracle (first and last client
        unless given), and every client decrypts."""
        got = self.matrix.computeResponses(np.stack([c["cts"] for c in clients]), self.dims, [c["key"] for c in clients])
        oracle_clients = {0, len(clients) - 1} if oracle_clients is None else oracle_clients
        for j, c in enumerate(clients):
            single = self.matrix.mulTransposeMatrix(c["cts"], self.dims, c["key"], modSwitchDownToSingle=True)
            assert got.shape[1:] == single.shape, (got.shape, single.shape)
            assert np.array_equal(got[j], single), f"client {j} differs from the single-client call"
            if j in oracle_clients:
                expected = self.oracle(c)
                assert len(expected) == got.shape[1]
                for i, ct in enumerate(expected):
                    assert np.array_equal(got[j, i], ct), (j, i)
            self.assert_decrypts(c, got[j], f"client {j}")
        return got

    def raw(self, keys, cts, capacity=None, matrix=None, count=None):
        """hecuda_pnns_compute_response_clients with raw handles; returns (rc, out, out_count)."""
        d = self.matrix._rowDescriptors(self.dims, cts.shape[1], self.elements)
        capacity = d["capacity"] if capacity is None else capacity
        count = len(keys) if count is None else count
        out = np.full((max(len(keys), 1), max(capacity, 1), 2, 1, self.n), 7, dtype=np.uint64)
        produced = C.c_int64(-1)
        handles = (C.c_void_p * max(len(keys), 1))(*[k._h for k in keys])
        rc = hecuda.load_library().hecuda_pnns_compute_response_clients(
            self.g._h, handles, count, (matrix or self.matrix)._h, np.ascontiguousarray(cts).ctypes.data_as(C.c_void_p),
            cts.shape[1], self.queries, d["index"], d["masks"].ctypes.data_as(C.c_void_p), d["rotate"], d["step"], d["plan"],
            d["planCount"], out.ctypes.data_as(C.c_void_p), capacity, C.byref(produced))
        return rc, out, produced.value

    def close(self, clients):
        for c in clients:
            c["key"].close()
        self.matrix.close()
        self.g.close()


MATRIX_SHAPES = [  # the shapes of test_gpu_pnns.py::test_mul_transpose_matrix_matches_oracle_and_decrypts
    (16, 1153, TEST_BITS, 4, 2, 3), (16, 1153, TEST_BITS, 3, 4, 5), (16, 1153, TEST_BITS, 8, 4, 2),
    (16, 1153, TEST_BITS, 20, 3, 3), (64, 65537, (55, 55, 55), 10, 8, 9), (64, 65537, (55, 55, 55), 40, 12, 4),
    (64, 65537, (55, 55, 55), 5, 32, 3), (64, 65537, (55, 55, 55), 10, 8, 1)]


@pytest.mark.parametrize("n,t,bits,rows,cols,queries", MATRIX_SHAPES + [
    (4096, 65537, (36, 36, 37), 300, 128, 20), (8192, 65537, (55, 55, 55, 55), 5000, 384, 3)])
def test_clients_match_single_client_and_oracle(n, t, bits, rows, cols, queries):
    s = Server(n, t, bits, rows, cols, queries, seed=rows * 131 + cols * 7 + queries)
    clients = [s.client(10 + j) for j in range(3 if n <= 64 else 2)]
    s.check(clients)
    s.close(clients)


@pytest.mark.parametrize("n,t,bits,rows,cols,queries", [(16, 1153, TEST_BITS, 4, 2, 3), (64, 65537, (55, 55, 55), 10, 8, 9)])
@pytest.mark.parametrize("count", [1, 2, GROUP, GROUP + 1, 2 * GROUP + 1])
def test_client_counts(count, n, t, bits, rows, cols, queries):
    s = Server(n, t, bits, rows, cols, queries, seed=count)
    clients = [s.client(200 + j) for j in range(count)]
    s.check(clients)
    s.close(clients)


@pytest.mark.parametrize("n,t,bits,rows,cols,queries", [(16, 1153, TEST_BITS, 4, 2, 3), (64, 65537, (55, 55, 55), 10, 8, 1),
                                                         (64, 65537, (55, 55, 55), 40, 12, 4)])
def test_wire_replies_match_oracle_and_decrypt(n, t, bits, rows, cols, queries):
    """Keys from EvaluationKey.fromSerialized, seeded queries in, replies serialized with skipLSBsForDecryption out."""
    s = Server(n, t, bits, rows, cols, queries, seed=n + rows)
    o, q0 = s.o, s.o.q[:1]
    rng = np.random.default_rng(n + rows)
    clients = []
    for j in range(3):
        sk, _, _, okeys, wire = seeded_keys(o, 300 + j, rng, s.elements, 7000 + 31 * j)
        key = hecuda.EvaluationKey.fromSerialized(s.g, galois=wire)
        query, cts = s.query(300 + j, sk)
        seeds = ref.random_seeds(rng, len(cts))
        seeded, poly0 = ref.reseed_query(o, sk, cts, seeds)
        clients.append(dict(sk=sk, key=key, okeys=okeys, query=query, cts=seeded, poly0=poly0, seeds=seeds))
    replies, skips = pnns.PnnsWire.computeResponses(s.matrix, np.stack([c["poly0"] for c in clients]),
                                                    np.stack([c["seeds"] for c in clients]), s.dims,
                                                    [c["key"] for c in clients])
    assert skips == opir.skip_lsbs_for_decryption(n, q0[0], t)
    half = opir.serialization_byte_count(n, q0, skips[0])
    assert replies.shape[2] == half + opir.serialization_byte_count(n, q0, skips[1])
    words = s.check(clients)  # the seeded ciphertexts as words: single-client and oracle parity, decryption
    assert replies.shape[:2] == words.shape[:2]
    for j, c in enumerate(clients):
        expected = s.oracle(c) if j in (0, len(clients) - 1) else list(words[j])
        recovered = []
        for i, ct in enumerate(expected):
            want = opir.serialize_poly(n, q0, ct[0], skips[0]) + opir.serialize_poly(n, q0, ct[1], skips[1])
            assert replies[j, i].tobytes() == want, (j, i)
            recovered.append(np.stack([opir.load_poly(n, q0, replies[j, i, :half].tobytes(), skips[0]),
                                       opir.load_poly(n, q0, replies[j, i, half:].tobytes(), skips[1])]))
        s.assert_decrypts(c, recovered, f"client {j} from its reply bytes")
    s.close(clients)


@pytest.mark.parametrize("queries", [1, 3])
def test_launch_counts(queries):
    """One client issues the launches of mulTransposeMatrix(modSwitchDownToSingle); from two clients up the launch count
    does not depend on the group's size."""
    s = Server(16, 1153, TEST_BITS, 4, 2, queries, seed=queries)
    clients = [s.client(400 + j) for j in range(GROUP)]
    cts = np.stack([c["cts"] for c in clients])
    keys = [c["key"] for c in clients]

    def launches(fn):
        before = hecuda.kernel_launch_count()
        fn()
        return hecuda.kernel_launch_count() - before

    single = launches(lambda: s.matrix.mulTransposeMatrix(cts[0], s.dims, keys[0], modSwitchDownToSingle=True))
    assert launches(lambda: s.matrix.computeResponses(cts[:1], s.dims, keys[:1])) == single
    two = launches(lambda: s.matrix.computeResponses(cts[:2], s.dims, keys[:2]))
    assert launches(lambda: s.matrix.computeResponses(cts, s.dims, keys)) == two
    assert launches(lambda: s.matrix.computeResponses(cts[:5], s.dims, keys[:5])) == two
    s.close(clients)


def test_errors_are_found_before_anything_is_enqueued():
    s = Server(16, 1153, TEST_BITS, 4, 2, 3, seed=5)
    swap = orc.galois_element_swapping_rows(16)
    assert swap in s.elements
    count, faulty = 20, 17
    clients = [s.client(500 + j) for j in range(count - 1)]
    clients.insert(faulty, s.client(600, elements=[e for e in s.elements if e != swap]))
    cts = np.stack([c["cts"] for c in clients])
    keys = [c["key"] for c in clients]
    before = hecuda.kernel_launch_count()
    rc, out, _ = s.raw(keys, cts)
    assert rc == ERR_MISSING_KEY
    message = hecuda.load_library().hecuda_last_error().decode()
    assert message.startswith(f"client {faulty}: ") and "missingGaloisElement" in message, message
    assert hecuda.kernel_launch_count() == before
    assert bool((out == 7).all()), "a failed call wrote replies"
    with pytest.raises(hecuda.HeError) as err:
        s.matrix.computeResponses(cts, s.dims, keys)
    assert err.value.code == ERR_MISSING_KEY and f"client {faulty}" in str(err.value)
    good = keys[:3]
    # a key of another context
    other = hecuda.Context(16, s.g.coefficientModuli, 1153)
    foreign = hecuda.EvaluationKey(other, None)
    with pytest.raises(hecuda.HeError) as err:
        s.matrix.computeResponses(cts[:3], s.dims, [good[0], foreign, good[2]])
    assert err.value.code == ERR_INVALID_ARGUMENT and "client 1: " in str(err.value)
    # a matrix of another context
    other_matrix = pnns.PlaintextMatrix(other, pnns.MatrixDimensions(s.rows, s.cols), s.flat)
    rc, out, _ = s.raw(good, cts[:3], matrix=other_matrix)
    assert rc == ERR_INVALID_ARGUMENT and bool((out == 7).all())
    other_matrix.close()
    foreign.close()
    other.close()
    # no clients
    rc, _, _ = s.raw(good, cts[:3], count=0)
    assert rc == ERR_INVALID_ARGUMENT
    # too small an output buffer: the count needed is reported
    needed = len(s.matrix.mulTransposeMatrix(cts[0], s.dims, good[0], modSwitchDownToSingle=True))
    before = hecuda.kernel_launch_count()
    rc, out, produced = s.raw(good, cts[:3], capacity=needed - 1)
    assert rc == ERR_INVALID_ARGUMENT and produced == needed and bool((out == 7).all())
    assert hecuda.kernel_launch_count() == before
    # a skip the reply modulus cannot drop
    d = s.matrix._rowDescriptors(s.dims, cts.shape[1], s.elements)
    size = hecuda.Bfv.serializationByteCount(s.g, s.g.L)
    poly0 = np.zeros((3, cts.shape[1], size), dtype=np.uint8)
    seeds = np.zeros((3, cts.shape[1], 32), dtype=np.uint8)
    handles = (C.c_void_p * 3)(*[k._h for k in good])
    wire_out = np.full((3, d["capacity"], 64), 7, dtype=np.uint8)
    produced = C.c_int64(0)
    rc = hecuda.load_library().hecuda_pnns_compute_response_clients_wire(
        s.g._h, handles, 3, s.matrix._h, poly0.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p), cts.shape[1],
        s.queries, d["index"], d["masks"].ctypes.data_as(C.c_void_p), d["rotate"], d["step"], d["plan"], d["planCount"], 200, 0,
        wire_out.ctypes.data_as(C.c_void_p), d["capacity"], C.byref(produced))
    assert rc == ERR_INVALID_ARGUMENT and bool((wire_out == 7).all())
    s.close(clients)


def test_concurrent_callers():
    """Two host threads answer different clients on the same matrix at once; each gets the sequential result."""
    s = Server(64, 65537, (55, 55, 55), 10, 8, 9, seed=11)
    clients = [s.client(700 + j) for j in range(6)]
    cts = np.stack([c["cts"] for c in clients])
    keys = [c["key"] for c in clients]
    halves = [[0, 1, 2], [3, 4, 5]]
    want = [s.matrix.computeResponses(cts[h], s.dims, [keys[i] for i in h]) for h in halves]
    results, errors = {}, []

    def worker(tid):
        try:
            for _ in range(3):
                h = halves[tid]
                results[tid] = s.matrix.computeResponses(cts[h], s.dims, [keys[i] for i in h])
                assert np.array_equal(results[tid], want[tid])
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    s.close(clients)
