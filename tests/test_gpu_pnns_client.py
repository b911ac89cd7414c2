"""The PNNS client on the GPU: float vectors normalised on the device, encrypted .denseRow queries, decrypted float
distances with the plaintext CRT, ProcessedDatabase.processOnDevice / validate and hecuda_evk_copy -- bit-exact against
tests/pnns_client_ref.py, and the reference's ClientTests run through hecuda.pnns."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pnns
from oracle import client_oracle as co
from oracle import oracle as orc

import pnns_client_ref as ref

OK, INVALID = 0, -1  # HECUDA_OK, HECUDA_ERR_INVALID_ARGUMENT
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]  # 4 x 55 bits (C5)


def seeds(tag, count):
    return np.frombuffer(b"".join(hashlib.sha256(repr((tag, i)).encode()).digest() for i in range(count)),
                         dtype=np.uint8).reshape(count, 32).copy()


def read_device(ptr, nbytes):
    import torch

    class Buffer:
        __cuda_array_interface__ = {"shape": (nbytes // 8,), "typestr": "<i8", "data": (ptr, False), "version": 2}

    return torch.as_tensor(Buffer(), device="cuda").cpu().numpy().view(np.uint64)


def contexts(n, moduli, ts):
    return [hecuda.Context(n, moduli, t) for t in ts], [orc.Context(n, moduli, t) for t in ts]


def config_for(n, moduli, ts, rows, cols, queries, s=None):
    params = pnns.EncryptionParameters(n, ts[0], tuple(moduli))
    s = pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, cols, ts) if s is None else s
    ekc = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(rows, cols), queries, n)
    cc = pnns.ClientConfig(params, s, cols, ekc, extraPlaintextModuli=ts[1:])
    return cc, pnns.ServerConfig(cc)


def database(vectors):
    return pnns.Database([pnns.DatabaseRow(i, bytes([i % 255]), list(v)) for i, v in enumerate(vectors)])


# ------------------------------------------------------------------------------------------------ signed values
@pytest.mark.parametrize("n,rows,cols", [(64, 65, 16), (64, 7, 3), (4096, 300, 128), (8192, 100000, 512)])
def test_signed_values_from_floats_bit_exact(n, rows, cols):
    t = orc.generate_primes([17], True, n)[0]
    moduli = orc.generate_primes([55, 55, 55], False, n)
    g = hecuda.Context(n, moduli, t)
    rng = np.random.default_rng(rows)
    vectors = rng.standard_normal((rows, cols)).astype(np.float32)
    vectors[rows // 2] = 0                                           # a zero row
    vectors[1, 0] = 1e20                                             # a large magnitude: the row's norm overflows to inf
    vectors[2] *= np.float32(1e-40)                                  # subnormal values: their squares vanish
    s = pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, cols, [t])
    expected = ref.normalized_scaled_and_rounded_array(vectors, s)
    cc, sc = config_for(n, moduli, [t], rows, cols, 1, s)
    db = pnns.Database([pnns.DatabaseRow(i, b"", v) for i, v in enumerate(vectors)])
    processed = pnns.ProcessedDatabase.processOnDevice(db, sc, [g])
    reference = pnns.PlaintextMatrix.fromSignedValues(g, pnns.MatrixDimensions(rows, cols), expected,
                                                      sc.babyStepGiantStep)
    got = read_device(*processed.plaintextMatrices[0].deviceBuffer())
    assert np.array_equal(got, read_device(*reference.deviceBuffer()))
    assert np.array_equal(processed.plaintextMatrices[0].presentFlags(), reference.presentFlags())
    reference.close()
    processed.close()


# ------------------------------------------------------------------------------------------------ queries
@pytest.mark.parametrize("n,rows,cols,extra", [(64, 3, 16, 0), (64, 9, 5, 1), (4096, 16, 128, 1), (8192, 16, 512, 0)])
def test_query_ciphertexts_bit_exact_full_and_seeded(n, rows, cols, extra):
    ts = orc.generate_primes([17] * (1 + extra), True, n)
    moduli = orc.generate_primes([55, 55, 55], False, n)
    gs, os_ = contexts(n, moduli, ts)
    cc, _ = config_for(n, moduli, ts, 100, cols, rows)
    client = pnns.Client(cc, gs)
    sk = client.generateSecretKey(seeds("sk", 1)[0])
    rng = np.random.default_rng(n + rows)
    vectors = rng.standard_normal((rows, cols)).astype(np.float32)
    count = pnns.CiphertextMatrix.ciphertextCount(n, pnns.MatrixDimensions(rows, cols))
    a = [seeds(("a", k), count) for k in range(len(ts))]
    e = [seeds(("e", k), count) for k in range(len(ts))]
    full = client.generateQuery(vectors, sk, aSeeds=a, errorSeeds=e)
    wire = client.generateQuery(vectors, sk, wire=True, aSeeds=a, errorSeeds=e)
    expected = ref.generate_query(os_, sk.poly, vectors.tolist(), cc.scalingFactor,
                                  [[bytes(x) for x in ak] for ak in a], [[bytes(x) for x in ek] for ek in e])
    for k, g in enumerate(gs):
        assert np.array_equal(full.ciphertextMatrices[k], expected[k]), k
        poly0, sd = wire.ciphertextMatrices[k]
        assert np.array_equal(hecuda.Bfv.expandSeeded(g, poly0, sd), expected[k]), k


def test_query_refusals_launch_nothing():
    n = 64
    t = orc.generate_primes([17], True, n)[0]
    g = hecuda.Context(n, orc.generate_primes([55, 55, 55], False, n), t)
    sk = hecuda.SecretKey.generate(g, seeds("sk", 1)[0])
    lib = hecuda.load_library()
    out = np.zeros((1, 2, g.L, n), dtype=np.uint64)
    a, e = seeds("a", 1), seeds("e", 1)

    def call(vectors, rows, cols, s, reduce=0):
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        before = hecuda.kernel_launch_count()
        rc = lib.hecuda_pnns_query_generate(g._h, sk.poly.ctypes.data, v.ctypes.data, rows, cols, s, reduce,
                                            a.ctypes.data, e.ctypes.data, out.ctypes.data, None)
        return rc, hecuda.kernel_launch_count() - before

    good = np.ones((1, 8), dtype=np.float32)
    assert call(good, 1, 8, 100)[0] == OK
    for v in (np.inf, -np.inf, np.nan):
        bad = good.copy()
        bad[0, 3] = v
        assert call(bad, 1, 8, 100) == (INVALID, 0), v
    assert call(np.ones((1, 40), dtype=np.float32), 1, 40, 100) == (INVALID, 0)  # > N/2 columns
    assert call(good, 1, 8, t) == (INVALID, 0)          # leaves [-t/2, t/2)
    assert call(good, 1, 8, 2 ** 62 + 2 ** 40, 1) == (INVALID, 0)  # leaves Int64


# ------------------------------------------------------------------------------------------------ distances
@pytest.mark.parametrize("moduli_count", [1, 2, 3])
@pytest.mark.parametrize("n,rows,cols,queries", [(64, 65, 16, 3), (64, 20, 8, 5), (4096, 3000, 128, 4)])
def test_distances_match_oracle_on_server_replies(n, rows, cols, queries, moduli_count):
    ts = orc.generate_primes([17, 18, 19][:moduli_count], True, n)
    moduli = orc.generate_primes([55, 55, 55, 55], False, n)
    gs, os_ = contexts(n, moduli, ts)
    cc, sc = config_for(n, moduli, ts, rows, cols, queries)
    rng = np.random.default_rng(rows * moduli_count)
    vectors = rng.standard_normal((rows, cols)).astype(np.float32)
    processed = pnns.ProcessedDatabase.processOnDevice(database(vectors), sc, gs)
    client, server = pnns.Client(cc, gs), pnns.Server(processed)
    sk = client.generateSecretKey()
    key = client.generateEvaluationKey(sk)
    query = client.generateQuery(vectors[:queries], sk)
    response = server.computeResponse(query, key)
    got = client.decrypt(response, sk)
    assert got.distances.shape == (rows, queries) and got.distances.dtype == np.float32
    expected = ref.decrypt(os_, sk.poly, [list(m) for m in response.ciphertextMatrices], rows, queries, cc.scalingFactor)
    assert np.array_equal(got.distances.view(np.uint32), expected.view(np.uint32))
    assert got.entryIds == list(range(rows))
    values = ref.normalized_scaled_and_rounded_array(vectors, cc.scalingFactor)
    product = math.prod(ts)
    exact = ref.mul_mod(values.tolist(), values[:queries].T.tolist(), product)
    assert np.array_equal(got.distances, ref.distances_from_signed(exact, cc.scalingFactor))
    key.close()
    processed.close()


def test_distance_refusals():
    n = 64
    moduli = orc.generate_primes([55, 55, 55], False, n)
    big = orc.generate_primes([31, 31, 31], True, n)          # 2 prod t > 2^64
    gs = [hecuda.Context(n, moduli, t) for t in big]
    sk = hecuda.SecretKey.generate(gs[0], seeds("sk", 1)[0])
    lib = hecuda.load_library()
    reply = np.zeros((1, 2, 1, n), dtype=np.uint64)
    out = np.zeros((4, 1), dtype=np.float32)

    def call(ctxs):
        hs = (C.c_void_p * len(ctxs))(*[c._h.value for c in ctxs])
        rs = (C.c_void_p * len(ctxs))(*[reply.ctypes.data] * len(ctxs))
        before = hecuda.kernel_launch_count()
        rc = lib.hecuda_pnns_decrypt_distances(hs, len(ctxs), sk.poly.ctypes.data, rs, 1, 1, 4, 1, 100, out.ctypes.data)
        return rc, hecuda.kernel_launch_count() - before

    assert call(gs[:2])[0] == OK                                                  # 2 prod t < 2^64
    assert call(gs) == (INVALID, 0)                      # 2 prod t > UInt64.max
    assert "UInt64.max" in hecuda.load_library().hecuda_last_error().decode()
    twin = hecuda.Context(n, moduli, big[0])
    assert call([gs[0], twin]) == (INVALID, 0)           # moduli not distinct
    other = hecuda.Context(n, orc.generate_primes([50, 50, 50], False, n), big[1])
    assert call([gs[0], other]) == (INVALID, 0)          # contexts differ in q


# ------------------------------------------------------------------------------------------------ reference cases
@pytest.mark.parametrize("extra", [False, True])
def test_query_as_response(extra):
    n, cols, s = 512, 32, 100
    ts = orc.generate_primes([16], True, n) + (orc.generate_primes([17], True, n) if extra else [])
    moduli = orc.generate_primes([27, 28, 28], False, n)
    gs, _ = contexts(n, moduli, ts)
    cc = pnns.ClientConfig(pnns.EncryptionParameters(n, ts[0], tuple(moduli)), s, cols, None, extraPlaintextModuli=ts[1:])
    client = pnns.Client(cc, gs)
    sk = client.generateSecretKey()
    values = np.array([[float((1 + c) % ts[0]) for c in range(cols)]], dtype=np.float32)
    query = client.generateQuery(values, sk)
    assert len(query.ciphertextMatrices) == len(ts)
    # the query as the response: a one-row .denseRow matrix reads as a 1 x cols .denseColumn matrix
    response = pnns.Response(query.ciphertextMatrices, pnns.MatrixDimensions(1, cols), [42], [(42).to_bytes(8, "little")])
    got = client.decrypt(response, sk)
    assert got.entryIds == [42] and got.entryMetadatas == [(42).to_bytes(8, "little")]
    expected = ref.distances_from_signed(ref.normalized_scaled_and_rounded(values.tolist(), s), s)
    assert np.array_equal(got.distances, expected)


@pytest.mark.parametrize("moduli_count", [1, 2])
@pytest.mark.parametrize("rows", [32, 64, 65, 192])
def test_client_server(rows, moduli_count):
    n, cols = 64, 16
    ts = orc.generate_primes([10] * 2, True, n)[:moduli_count]
    moduli = orc.generate_primes([60] * 3, False, n)
    gs, _ = contexts(n, moduli, ts)
    cc, sc = config_for(n, moduli, ts, rows, cols, 1)
    db = ref.database_for_testing(rows, cols)
    processed = pnns.ProcessedDatabase.processOnDevice(
        pnns.Database([pnns.DatabaseRow(i, m, v) for i, m, v in db]), sc, gs)
    client, server = pnns.Client(cc, processed.contexts), pnns.Server(processed)
    query_vectors = np.array([db[0][2]], dtype=np.float32)
    sk = client.generateSecretKey()
    query = client.generateQuery(query_vectors, sk)
    key = client.generateEvaluationKey(sk)
    response = server.computeResponse(query, key)
    assert response.noiseBudget(gs, sk) > 0
    got = client.decrypt(response, sk)
    assert got.entryIds == processed.entryIds and got.entryMetadatas == processed.entryMetadatas
    expected = ref.fixed_point_cosine_similarity([v for _, _, v in db], query_vectors.T.tolist(), math.prod(ts),
                                                 cc.scalingFactor)
    assert np.array_equal(got.distances, expected)
    key.close()
    processed.close()


# ------------------------------------------------------------------------------------------------ C5 shape
@pytest.fixture(scope="module", params=[0, 1], ids=["one-modulus", "extra-modulus"])
def c5(request):
    n, rows, cols, queries = 8192, 2000, 512, 16
    ts = [65537] + [t for t in orc.generate_primes([17, 17], True, n) if t != 65537][:request.param]
    gs, os_ = contexts(n, Q8192, ts)
    cc, sc = config_for(n, Q8192, ts, rows, cols, queries)
    rng = np.random.default_rng(55 + request.param)
    vectors = rng.standard_normal((rows, cols)).astype(np.float32)
    processed = pnns.ProcessedDatabase.processOnDevice(database(vectors), sc, gs)
    yield dict(gs=gs, os=os_, cc=cc, processed=processed, vectors=vectors, queries=queries, ts=ts)
    processed.close()


def test_c5_end_to_end_self_distances(c5):
    cc, processed, vectors, q = c5["cc"], c5["processed"], c5["vectors"], c5["queries"]
    client, server = pnns.Client(cc, c5["gs"]), pnns.Server(processed)
    sk = client.generateSecretKey()
    key = client.generateEvaluationKey(sk)
    response = server.computeResponse(client.generateQuery(vectors[:q], sk), key)
    got = client.decrypt(response, sk).distances
    assert got.shape == (len(vectors), q)
    for r in range(q):
        assert abs(got[r, r] - 1.0) <= 0.01, (r, got[r, r])     # PNNSProcessDatabase's trialDistanceTolerance
    key.close()


def test_c5_many_clients_match_single_calls(c5):
    cc, processed, vectors, q = c5["cc"], c5["processed"], c5["vectors"], c5["queries"]
    client, server = pnns.Client(cc, c5["gs"]), pnns.Server(processed)
    keys, queries, wires, sks = [], [], [], []
    for c in range(3):
        sk = client.generateSecretKey()
        sks.append(sk)
        keys.append(client.generateEvaluationKey(sk))
        queries.append(client.generateQuery(vectors[c:c + q], sk))
        wires.append(client.generateQuery(vectors[c:c + q], sk, wire=True))
    many = server.computeResponses(queries, keys)
    many_wire = server.computeResponses(wires, keys)
    for c in range(3):
        single = server.computeResponse(queries[c], keys[c])
        for k in range(len(c5["gs"])):
            assert np.array_equal(many[c].ciphertextMatrices[k], single.ciphertextMatrices[k]), (c, k)
        a = client.decrypt(single, sks[c]).distances
        assert np.array_equal(client.decrypt(many_wire[c], sks[c]).distances, a), c
    for k in keys:
        k.close()


# ------------------------------------------------------------------------------------------------ validate
def test_validate_noise_budget_equals_oracle(c5, monkeypatch):
    processed = c5["processed"]
    secret_keys = []
    generate = pnns.Client.generateSecretKey

    def recording(self, seed=None):   # keep each trial's secret key to recompute its budget on the CPU
        secret_keys.append(generate(self, seed))
        return secret_keys[-1]

    monkeypatch.setattr(pnns.Client, "generateSecretKey", recording)
    result = processed.validate(c5["vectors"][:c5["queries"]], trials=2)
    assert len(result.computeTimes) == 2 and len(secret_keys) == 2
    distances = result.databaseDistances.distances
    assert distances.shape == (len(c5["vectors"]), c5["queries"])
    for r in range(c5["queries"]):
        assert abs(distances[r, r] - 1.0) <= 0.01
    # the returned response is the last trial's
    last = min(co.noise_budget(8192, Q8192, o.t, secret_keys[-1].poly, ct)
               for o, m in zip(c5["os"], result.response.ciphertextMatrices) for ct in m)
    assert result.response.noiseBudget(c5["gs"], secret_keys[-1]) == last
    assert result.noiseBudget <= last and result.noiseBudget > hecuda.Bfv.minNoiseBudget
    result.evaluationKey.close()


def test_validate_errors(monkeypatch):
    n, rows, cols = 64, 20, 16
    ts = orc.generate_primes([10], True, n)
    moduli = orc.generate_primes([60, 60, 60], False, n)
    gs, os_ = contexts(n, moduli, ts)
    cc, sc = config_for(n, moduli, ts, rows, cols, 1)
    vectors = np.random.default_rng(3).standard_normal((rows, cols)).astype(np.float32)
    processed = pnns.ProcessedDatabase.processOnDevice(database(vectors), sc, gs)
    with pytest.raises(pnns.PnnsError, match="Invalid trialsPerShard: 0"):
        processed.validate(vectors[:1], trials=0)
    with pytest.raises(pnns.PnnsError, match="Wrong vector dimension 15, expected 16"):
        processed.validate(vectors[:1, :15])
    # Bfv.minNoiseBudget is 0 and a centred norm never exceeds q / 2, so a BFV budget is never below it: raise the
    # minimum above the response's real budget to reach the check, and record what the trial did
    seen = {"keys": [], "responses": [], "decrypted": 0}
    generate, respond = pnns.Client.generateSecretKey, pnns.Server.computeResponse

    def keep_key(self, seed=None):
        seen["keys"].append(generate(self, seed))
        return seen["keys"][-1]

    def keep_response(self, query, key):
        seen["responses"].append(respond(self, query, key))
        return seen["responses"][-1]

    def count_decrypt(self, response, secretKey):
        seen["decrypted"] += 1

    monkeypatch.setattr(pnns.Client, "generateSecretKey", keep_key)
    monkeypatch.setattr(pnns.Server, "computeResponse", keep_response)
    monkeypatch.setattr(pnns.Client, "decrypt", count_decrypt)
    monkeypatch.setattr(hecuda.Bfv, "minNoiseBudget", 1000.0)
    with pytest.raises(pnns.PnnsError, match="Insufficient noise budget"):
        processed.validate(vectors[:1])
    oracle = min(co.noise_budget(n, moduli, ts[0], seen["keys"][0].poly, ct) for ct in seen["responses"][0].ciphertextMatrices[0])
    assert oracle < hecuda.Bfv.minNoiseBudget
    assert seen["decrypted"] == 0                    # the budget is checked before decryption, as the reference does
    processed.close()


# ------------------------------------------------------------------------------------------------ evk copy
def test_evk_copy_words_lifetime_and_refusals():
    n = 4096
    moduli = orc.generate_primes([36, 36, 37], False, n)
    ts = orc.generate_primes([17, 18], True, n)
    g0, g1 = hecuda.Context(n, moduli, ts[0]), hecuda.Context(n, moduli, ts[1])
    sk = hecuda.SecretKey.generate(g0, seeds("sk", 1)[0])
    config = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(100, 64), 4, n)
    key = hecuda.EvaluationKey.generate(g0, config, sk)
    copy = key.forContext(g1)
    assert copy is key.forContext(g1) and key.forContext(g0) is key
    assert np.array_equal(read_device(*copy.deviceBuffer()), read_device(*key.deviceBuffer()))
    words = {e: read_device(*key.galoisDeviceBuffer(e)) for e in config.galoisElements}
    for e in config.galoisElements:
        assert np.array_equal(read_device(*copy.galoisDeviceBuffer(e)), words[e]), e
    # the copy outlives its source
    h = C.c_void_p()
    lib = hecuda.load_library()
    assert lib.hecuda_evk_copy(key._h, g1._h, C.byref(h)) == OK
    standalone = hecuda.EvaluationKey.__new__(hecuda.EvaluationKey)
    standalone.context, standalone.galoisElements, standalone._h = g1, list(config.galoisElements), h
    key.close()
    for e in config.galoisElements:
        assert np.array_equal(read_device(*standalone.galoisDeviceBuffer(e)), words[e]), e
    standalone.close()
    # refusals: different N, different moduli, different word size; *out NULL, nothing launched
    key = hecuda.EvaluationKey.generate(g0, config, sk)
    others = [hecuda.Context(2 * n, orc.generate_primes([36, 36, 37], False, 2 * n), orc.generate_primes([17], True, 2 * n)[0]),
              hecuda.Context(n, orc.generate_primes([36, 36, 36], False, n), ts[0]),
              hecuda.Context(n, orc.generate_primes([28, 28, 28], False, n), ts[0], scalar=np.uint32)]
    key32 = hecuda.EvaluationKey(others[2], None)
    for other, src in [(others[0], key), (others[1], key), (others[2], key), (g0, key32)]:
        h = C.c_void_p(12345)
        before = hecuda.kernel_launch_count()
        assert lib.hecuda_evk_copy(src._h, other._h, C.byref(h)) == INVALID
        assert h.value is None and hecuda.kernel_launch_count() == before
    key32.close()
    key.close()
