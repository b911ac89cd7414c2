"""PNNS requests and responses in the reference's protobuf messages on the GPU
(hecuda_pnns_compute_response_clients_proto): PNNSRequest in, PNNSShardResponse out, every plaintext modulus in one call.

- Byte parity: every client's PNNSShardResponse equals tests/pnns_proto_ref.py's framing around the replies
  hecuda_pnns_compute_response_clients_wire returns for the same poly0 and seeds, with keys copied per context by
  EvaluationKey.forContext and the row descriptors of PlaintextMatrix._rowDescriptors.  At the C5 shape with one-vector
  clients, and at N = 64 with multi-row queries against a database short enough that the packing rotations and
  swapRows run; for 1, 2, 16 and 17 clients, and with 1, 2 and 3 plaintext moduli.
- .full query ciphertexts answer like their seeded form.
- End to end: device clients send PNNSRequests with their keys inside; the server loads the keys from the request's
  ranges with EvaluationKey.fromProtoMany and answers with one call; every client decrypts what Client.decrypt of
  Server.computeResponses gives.
- Refusals name the client and leave the output untouched; the launch count of a group does not depend on its size."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
import pir_proto_ref as pref
import pnns_proto_ref as ref
from hecuda import pnns
from hecuda.pir import EvaluationKeyConfig
from oracle import oracle as orc

ERR_INVALID_ARGUMENT, ERR_MISSING_KEY = -1, -5
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]  # 4 x 55 bits (C5)


class Setup:
    """A processed database on one context per plaintext modulus, a client and a server of it."""

    def __init__(self, n, moduli, ts, rows, cols, queries, seed=0):
        self.n, self.moduli, self.ts, self.rows, self.cols, self.queries = n, moduli, ts, rows, cols, queries
        self.gs = [hecuda.Context(n, moduli, t) for t in ts]
        params = pnns.EncryptionParameters(n, ts[0], tuple(moduli))
        s = pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, cols, ts)
        ekc = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(rows, cols), queries, n)
        self.cc = pnns.ClientConfig(params, s, cols, ekc, extraPlaintextModuli=ts[1:])
        rng = np.random.default_rng(seed)
        self.vectors = rng.standard_normal((rows, cols)).astype(np.float32)
        db = pnns.Database([pnns.DatabaseRow(i * 7 + 1, bytes([i % 251]) * (i % 3), list(v))
                            for i, v in enumerate(self.vectors)])
        self.processed = pnns.ProcessedDatabase.processOnDevice(db, pnns.ServerConfig(self.cc), self.gs)
        self.client, self.server = pnns.Client(self.cc, self.gs), pnns.Server(self.processed)
        self.rng = rng

    def make_clients(self, count, with_key=False):
        out = []
        for j in range(count):
            sk = self.client.generateSecretKey()
            key, key_message = self.client.evaluationKeyMessage(sk)
            v = self.vectors[(j * self.queries) % self.rows:][:self.queries]
            if len(v) < self.queries:
                v = self.vectors[:self.queries]
            message = self.client.requestMessage(v, sk, evaluationKey=key_message if with_key else None,
                                                 keyTimestamp=100 + j, keyIdentifier=b"k%d" % j)
            out.append(dict(sk=sk, key=key, key_message=key_message, message=message, vectors=v))
        return out

    def query_sizes(self):
        return pref.poly_sizes(self.n, [q.bit_length() for q in self.moduli[:self.gs[0].L]])

    def seeded(self, message):
        """Per context: (poly0 (count, B), seeds (count, 32)) of a request, read by the restatement."""
        out = []
        for begin, end in ref.parse_pnns_request(message)["query"]:
            _, _, _, cts = ref.parse_matrix(message, begin, end, self.query_sizes())
            out.append((np.stack([np.frombuffer(ct[1], np.uint8) for ct in cts]),
                        np.stack([np.frombuffer(ct[2], np.uint8) for ct in cts])))
        return out

    def expected(self, cs):
        """The restatement's PNNSShardResponse around each client's _clients_wire replies, keys copied per context."""
        per_context = []
        seeded = [self.seeded(c["message"]) for c in cs]
        dims = pnns.MatrixDimensions(self.queries, self.cols)
        for k, m in enumerate(self.processed.plaintextMatrices):
            keys = [c["key"].forContext(m.context) for c in cs]
            replies, skips = pnns.PnnsWire.computeResponses(m, np.stack([s[k][0] for s in seeded]),
                                                            np.stack([s[k][1] for s in seeded]), dims, keys)
            b0 = hecuda.Bfv.serializationByteCount(m.context, 1, skips[0])
            per_context.append([([(r[:b0].tobytes(), r[b0:].tobytes()) for r in replies[j]], skips) for j in range(len(cs))])
        return [ref.encode_shard_response([per_context[k][j] for k in range(len(per_context))], self.rows, self.queries,
                                          self.processed.entryIds, self.processed.entryMetadatas) for j in range(len(cs))]

    def raw(self, messages, keys, capacity=1 << 22):
        """hecuda_pnns_compute_response_clients_proto into a filled buffer: (rc, error, buffer untouched)."""
        lib = hecuda.load_library()
        out = np.full(capacity, 0xAB, dtype=np.uint8)
        bufs = [np.frombuffer(m, np.uint8) if len(m) else np.zeros(1, np.uint8) for m in messages]
        counts = np.array([len(m) for m in messages], dtype=np.uint64)
        ms = self.processed.plaintextMatrices
        ids = np.asarray(self.processed.entryIds, dtype=np.uint64)
        meta = self.processed.entryMetadatas
        offsets = np.zeros(len(meta) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(x) for x in meta])
        blob = np.frombuffer(b"".join(meta) or b"\0", np.uint8)
        rc = lib.hecuda_pnns_compute_response_clients_proto(
            (C.c_void_p * len(ms))(*[m.context._h.value for m in ms]), len(ms),
            (C.c_void_p * len(keys))(*[k._h.value for k in keys]), len(keys),
            (C.c_void_p * len(ms))(*[m._h.value for m in ms]), (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs]),
            counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), ids.size, blob.ctypes.data_as(C.c_void_p),
            offsets.ctypes.data_as(C.c_void_p), len(meta), out.ctypes.data_as(C.c_void_p))
        return rc, lib.hecuda_last_error().decode() if rc else "", bool((out == 0xAB).all())

    def close(self, cs=()):
        for c in cs:
            c["key"].close()
        self.processed.close()


def small(ts_count, queries=5, rows=8):
    n = 64
    ts = orc.generate_primes([12] * 3, True, n)[:ts_count]
    return Setup(n, orc.generate_primes([60] * 3, False, n), ts, rows, 16, queries, seed=ts_count * 10 + queries)


@pytest.fixture(scope="module")
def c5():
    s = Setup(8192, Q8192, [65537], 100000, 512, 1, seed=5)
    yield s
    s.close()


@pytest.mark.parametrize("count", [1, 17])
def test_c5_parity_with_the_wire_path(c5, count):
    cs = c5.make_clients(count)
    got = c5.server.computeResponsesProto([c["message"] for c in cs], [c["key"] for c in cs])
    assert got == c5.expected(cs)
    for c in cs:
        c["key"].close()


@pytest.mark.parametrize("ts_count", [1, 2, 3])
@pytest.mark.parametrize("count", [1, 2, 16, 17])
def test_small_parity_with_the_wire_path(count, ts_count):
    """N = 64, 8 database rows: 4 query rows per SIMD row, so the packing rotations and swapRows run; 5-row queries."""
    if ts_count > 1 and count not in (2, 17):
        pytest.skip("the plaintext CRT runs at 2 and 17 clients")
    s = small(ts_count)
    cs = s.make_clients(count)
    got = s.server.computeResponsesProto([c["message"] for c in cs], [c["key"] for c in cs])
    assert got == s.expected(cs)
    s.close(cs)


def test_full_query_ciphertexts_answer_like_seeded():
    s = small(2)
    cs = s.make_clients(2)
    keys = [c["key"] for c in cs]
    full = []
    for j, c in enumerate(cs):
        matrices = []
        for k, (poly0, seeds) in enumerate(s.seeded(c["message"])):
            g = s.gs[k]
            polys = hecuda.Bfv.serialize(g, hecuda.Bfv.expandSeeded(g, poly0, seeds))
            skips = [0, 0] if j == 0 else []
            cts = [("full", pref.full_polys(polys[2 * i].tobytes(), polys[2 * i + 1].tobytes()), skips, 1)
                   for i in range(len(poly0))]
            matrices.append(ref.encode_matrix(s.queries, s.cols, cts, ref.DENSE_ROW))
        full.append(ref.encode_pnns_request(matrices))
    seeded = s.server.computeResponsesProto([c["message"] for c in cs], keys)
    assert s.server.computeResponsesProto(full, keys) == seeded
    assert s.server.computeResponsesProto([full[0], cs[1]["message"]], keys) == seeded
    s.close(cs)


@pytest.mark.parametrize("ts_count", [1, 2])
def test_end_to_end(ts_count):
    """16 clients send requests with their keys inside; the keys are loaded from the request's ranges in one call."""
    s = small(ts_count, queries=3, rows=12)
    cs = s.make_clients(16, with_key=True)
    messages = [c["message"] for c in cs]
    fields = [pnns.PnnsRequest.fields(m) for m in messages]
    for j, f in enumerate(fields):
        assert (f["queryCount"], f["queryRowCount"]) == (len(s.gs), s.queries)
        assert (f["keyTimestamp"], f["keyIdentifier"]) == (100 + j, b"k%d" % j)
        at, size = f["evaluationKey"]
        assert messages[j][at:at + size] == cs[j]["key_message"]
    keys = hecuda.EvaluationKey.fromProtoMany(s.gs[0], [m[f["evaluationKey"][0]:sum(f["evaluationKey"])]
                                                        for m, f in zip(messages, fields)])
    replies = s.server.computeResponsesProto(messages, keys)
    queries = [s.client.generateQuery(c["vectors"], c["sk"]) for c in cs]
    plain = s.server.computeResponses(queries, [c["key"] for c in cs])
    for j, c in enumerate(cs):
        got = s.client.decryptResponseMessage(replies[j], c["sk"])
        want = s.client.decrypt(plain[j], c["sk"])
        assert np.array_equal(got.distances, want.distances), j
        assert got.entryIds == s.processed.entryIds and got.entryMetadatas == s.processed.entryMetadatas
    for k in keys:
        k.close()
    s.close(cs)


def test_refusals_name_the_client_and_leave_out_untouched():
    s = small(2)
    cs = s.make_clients(3)
    keys = [c["key"] for c in cs]
    good = [c["message"] for c in cs]
    assert s.raw(good, keys)[0] == 0
    sizes = s.query_sizes()
    q = ref.parse_pnns_request(good[1])["query"]
    mats = [ref.parse_matrix(good[1], b, e, sizes) for b, e in q]
    rows, cols, _, cts = mats[0]

    def request(matrices):
        return ref.encode_pnns_request(matrices)

    one = ref.encode_matrix(rows, cols, cts, ref.DENSE_ROW)
    bad = {
        "wrongCiphertextMatrixCount": request([one]),
        "wrongMatrixPacking": request([ref.encode_matrix(rows, cols, cts, ref.DIAGONAL), one]),
        "unsetOneof": request([ref.encode_matrix(rows, cols, cts, None), one]),
        "invalidMatrixDimensions": request([ref.encode_matrix(rows, cols + 1, cts, ref.DENSE_ROW)] * 2),
        "wrongCiphertextCount": request([ref.encode_matrix(rows, cols, cts + cts, ref.DENSE_ROW), one]),
        "rows differ": request([ref.encode_matrix(rows - 1, cols, cts, ref.DENSE_ROW), one]),
        "client 0's rows": request([ref.encode_matrix(rows - 4, cols, cts[:1], ref.DENSE_ROW)] * 2),
        "short seed": request([ref.encode_matrix(rows, cols, [("seeded", cts[0][1], cts[0][2][:31])] + cts[1:],
                                                 ref.DENSE_ROW), one]),
        "truncated": good[1][:-1],
    }
    for name, message in bad.items():
        rc, err, untouched = s.raw([good[0], message, good[2]], keys)
        assert rc == ERR_INVALID_ARGUMENT, (name, rc, err)
        assert err.startswith("client 1: "), (name, err)
        assert untouched, name
    # a key of a context with other coefficient moduli
    other = hecuda.Context(s.n, orc.generate_primes([59] * 3, False, s.n), s.ts[0])
    sk = hecuda.SecretKey.generate(other)
    foreign = hecuda.EvaluationKey.generate(other, s.cc.evaluationKeyConfig, sk)
    rc, err, untouched = s.raw(good, [keys[0], foreign, keys[2]])
    assert rc == ERR_INVALID_ARGUMENT and err.startswith("client 1: invalidContext") and untouched, err
    # a key without one of the Galois elements the plan needs
    sk2 = s.client.generateSecretKey()
    elements = list(s.cc.evaluationKeyConfig.galoisElements)
    partial = hecuda.EvaluationKey.generate(s.gs[0], EvaluationKeyConfig(elements[:-1], False), sk2)
    rc, err, untouched = s.raw(good, [keys[0], keys[1], partial])
    assert rc == ERR_MISSING_KEY and err.startswith("client 2: ") and untouched, err
    foreign.close()
    partial.close()
    s.close(cs)


def test_launch_count_does_not_depend_on_the_group_size():
    s = small(2)
    cs = s.make_clients(16)
    messages, keys = [c["message"] for c in cs], [c["key"] for c in cs]

    def launches(count):
        before = hecuda.kernel_launch_count()
        s.server.computeResponsesProto(messages[:count], keys[:count])
        return hecuda.kernel_launch_count() - before

    two = launches(2)
    assert launches(5) == two
    assert launches(16) == two
    s.close(cs)
