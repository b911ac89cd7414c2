"""The symmetric-PIR OPRF server on the device: hecuda_oprf_blind_evaluate and hecuda.symmetric_pir.OprfServer
bit-exact against tests/oprf_proof_ref.py, the reference's oprfRoundtrip and roundTrip through OprfServer, a call past
the 65535-query launch split, invalid queries inside a batch, seeds, and the refusals."""
import multiprocessing
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda  # noqa: E402
import oprf_proof_ref as R  # noqa: E402
from hecuda import keyword_pir as kw  # noqa: E402
from hecuda import pir  # noqa: E402
from hecuda import symmetric_pir as sp  # noqa: E402
from oracle import oprf_oracle as O  # noqa: E402

ERR_INVALID_ARGUMENT = -1
KEY = random.Random(30).randrange(1, O.N).to_bytes(48, "big")
SEED = bytes(range(32))
P = hecuda._ptr


def invalid_queries():
    """Each kind of invalid encoding: prefixes 0, 1 and 4, x = p, x > p, x off the curve, all zeros."""
    good = O.blind(b"neighbour", 5)[1]
    off_curve = next(x for x in range(1, 100) if not O.is_square((x ** 3 + O.A * x + O.B) % O.P))
    return [bytes([0]) + good[1:], bytes([1]) + good[1:], bytes([4]) + good[1:], b"\x02" + O.P.to_bytes(48, "big"),
            b"\x03" + (O.P + 1).to_bytes(48, "big"), b"\x02" + off_curve.to_bytes(48, "big"), bytes(49)]


def blind_evaluate(lib, key, queries, seed=SEED):
    count = len(queries)
    blinded = np.frombuffer(b"".join(queries) or b"\0", dtype=np.uint8)
    responses = np.zeros((max(count, 1), 145), dtype=np.uint8)
    status = np.full(max(count, 1), 7, dtype=np.uint8)
    rc = lib.hecuda_oprf_blind_evaluate(P(np.frombuffer(key, dtype=np.uint8)), P(blinded), count,
                                         P(np.frombuffer(seed, dtype=np.uint8)), P(responses), P(status))
    assert rc == 0, (lib.hecuda_last_error() or b"").decode()
    return [r.tobytes() for r in responses[:count]], status[:count].tolist()


def _expected(args):
    data, blind_scalar, query = args
    response = R.blind_evaluate_verifiable(KEY, query, SEED)
    return response, R.finalize_verifiable(data, blind_scalar, response, O.public_key(KEY))


@pytest.fixture(scope="module")
def blinded():
    rng = random.Random(31)
    inputs = [rng.randbytes(rng.randrange(1, 40)) for _ in range(512)]
    blinds = [rng.randrange(1, O.N) for _ in inputs]
    queries = [O.blind(m, r)[1] for m, r in zip(inputs, blinds)]
    with multiprocessing.get_context("fork").Pool(8) as pool:
        expected = pool.map(_expected, list(zip(inputs, blinds, queries)))
    return inputs, blinds, queries, expected


def test_bit_exact_and_verifiable(blinded):
    """512 oracle-blinded queries: byte-equal to the restatement with status 0, and each response verifies and
    finalizes to hecuda_oprf_evaluate's output for the same input."""
    inputs, _, queries, expected = blinded
    responses, status = blind_evaluate(hecuda.load_library(), KEY, queries)
    assert status == [0] * len(queries)
    assert responses == [r for r, _ in expected]
    evaluated = sp.Oprf.evaluate(KEY, inputs)
    assert [bytes(h) for h in evaluated] == [h for _, h in expected]


def test_oprf_roundtrip():
    """SymmetricPIRTests.oprfRoundtrip: one keyword twice gives different queries and equal outputs."""
    config = sp.SymmetricPirConfig(KEY)
    server = sp.OprfServer(config)
    client = R.OprfClient(config.clientConfig().serverPublicKey)
    keyword = bytes([1, 2, 3, 4, 5])
    outputs, queries = [], []
    for _ in range(2):
        context = client.queryContext(keyword)
        queries.append(context[2])
        outputs.append(client.parse(server.computeResponse(context[2]), context))
    assert queries[0] != queries[1]
    assert outputs[0] == outputs[1]
    assert outputs[0][0] == O.evaluate(KEY, keyword)[:16]


@pytest.fixture(scope="module")
def test_context():
    import oracle.oracle as orc

    n, t = 16, 1153
    ctx = hecuda.Context(n, orc.generate_primes([55, 52, 62, 58], False, n), t)
    yield ctx
    ctx.close()


def round_trip(g, database, encrypted, config):
    """SymmetricPirTests.roundTrip (_TestUtilities/PirUtilities/SymmetricPirTests.swift:33-95): OPRF through OprfServer,
    keyword PIR at the oblivious keyword, then the AES-GCM open."""
    keyword_config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(100), True, "noCompression",
                                         symmetricPirClientConfig=config.clientConfig())
    processed = kw.KeywordPirServer.processOnDevice(encrypted, keyword_config, g, symmetricPirConfig=config)
    server = kw.KeywordPirServer(g, processed)
    client = kw.KeywordPirClient(keyword_config.parameter, processed.pirParameter, g)
    oprf_server = sp.OprfServer(config)
    oprf_client = R.OprfClient(keyword_config.symmetricPirClientConfig.serverPublicKey)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    indices = list(range(len(database)))
    random.Random(32).shuffle(indices)
    for index in indices[:10]:
        keyword, value = database[index]
        context = oprf_client.queryContext(keyword)
        parsed = oprf_client.parse(oprf_server.computeResponse(context[2]), context)
        response = server.computeResponse(client.generateQuery(parsed[0], sk), key)
        sealed = client.decrypt(response, parsed[0], sk)
        assert sealed is not None
        assert oprf_client.decrypt(sealed, parsed) == value
    key.close()
    processed.close()


def test_round_trip(test_context):
    g = test_context
    rng = random.Random(33)
    database = [(b"keyword %d" % i, rng.randbytes(pir.bytesPerPlaintext(g) // 2)) for i in range(100)]
    config = sp.SymmetricPirConfig(KEY)
    round_trip(g, database, kw.KeywordDatabase.symmetricPIRProcess(database, config), config)


def test_round_trip_through_sharding(test_context):
    g = test_context
    rng = random.Random(34)
    database = [(b"row %d" % i, rng.randbytes(pir.bytesPerPlaintext(g) // 2)) for i in range(200)]
    config = sp.SymmetricPirConfig(KEY)
    sharded = kw.KeywordDatabase(database, kw.Sharding.shardCount(2), symmetricPirConfig=config)
    plain = dict(database)
    reverse = {O.evaluate(KEY, k)[:16]: (k, plain[k]) for k in plain}
    for shard_rows in sharded.shards.values():
        round_trip(g, [reverse[k] for k, _ in shard_rows], shard_rows, config)


def test_past_the_launch_split():
    """70000 queries in one call equal the calls on [0, 65535) and [65535, 70000), and the restatement at both sides of
    the split; the call launches one more kernel of each per-query kind than a one-query call."""
    count = 70000
    base = [O.blind(b"split %d" % i, 1000 + i)[1] for i in range(64)]
    queries = [base[i % len(base)] for i in range(count)]
    lib = hecuda.load_library()
    before = hecuda.kernel_launch_count()
    blind_evaluate(lib, KEY, queries[:1])
    one = hecuda.kernel_launch_count() - before
    before = hecuda.kernel_launch_count()
    whole, status = blind_evaluate(lib, KEY, queries)
    assert hecuda.kernel_launch_count() - before == one + 2 == 5
    assert status == [0] * count
    first, _ = blind_evaluate(lib, KEY, queries[:65535])
    second, _ = blind_evaluate(lib, KEY, queries[65535:])
    assert whole == first + second
    for i in (0, 65534, 65535, 65536, 69999):
        assert whole[i] == R.blind_evaluate_verifiable(KEY, queries[i], SEED)


def test_invalid_queries_inside_a_batch():
    """Each kind of invalid query gets status 1 and zero bytes; its neighbours equal a batch without it."""
    lib = hecuda.load_library()
    good = [O.blind(b"good %d" % i, 77 + i)[1] for i in range(8)]
    bad = invalid_queries()
    mixed, where = [], []
    for i, b in enumerate(bad):
        mixed.append(good[i % len(good)])
        where.append(len(mixed))
        mixed.append(b)
    mixed.append(good[0])
    responses, status = blind_evaluate(lib, KEY, mixed)
    clean_responses, clean_status = blind_evaluate(lib, KEY, [q for i, q in enumerate(mixed) if i not in where])
    assert [status[i] for i in where] == [1] * len(bad)
    assert all(responses[i] == bytes(145) for i in where)
    assert [r for i, r in enumerate(responses) if i not in where] == clean_responses
    assert clean_status == [0] * len(clean_responses)
    server = sp.OprfServer(sp.SymmetricPirConfig(KEY))
    out = server.computeResponses([good[0], b"\x02" + bytes(10), bad[0], good[1]], SEED)
    assert out == [clean_responses[0], None, None, R.blind_evaluate_verifiable(KEY, good[1], SEED)]


def test_seeds():
    """The same seed gives the same response; another seed keeps the evaluated element and changes the proof, and both
    verify."""
    server = sp.OprfServer(sp.SymmetricPirConfig(KEY))
    data, blind_scalar = b"seeded", 12345
    query = O.blind(data, blind_scalar)[1]
    a = server.computeResponse(query, seed=bytes(32))
    assert a == server.computeResponse(query, seed=bytes(32))
    b = server.computeResponse(query, seed=b"\x01" * 32)
    assert a[:49] == b[:49] and a[49:] != b[49:]
    pk = O.public_key(KEY)
    assert R.finalize_verifiable(data, blind_scalar, a, pk) == R.finalize_verifiable(data, blind_scalar, b, pk) == \
        O.evaluate(KEY, data)
    assert len(server.computeResponse(query)) == 145  # a random seed


def refusal(call):
    lib = hecuda.load_library()
    before = hecuda.kernel_launch_count()
    rc = call(lib)
    message = (lib.hecuda_last_error() or b"").decode()
    assert hecuda.kernel_launch_count() == before
    return rc, message


@pytest.mark.parametrize("bad", [0, O.N, 2**384 - 1])
def test_bad_keys_are_refused(bad):
    key = np.frombuffer(bad.to_bytes(48, "big"), dtype=np.uint8)
    query = np.frombuffer(O.blind(b"k", 3)[1], dtype=np.uint8)
    seed, out, status = np.zeros(32, dtype=np.uint8), np.zeros(145, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
    rc, message = refusal(lambda lib: lib.hecuda_oprf_blind_evaluate(P(key), P(query), 1, P(seed), P(out), P(status)))
    assert rc == ERR_INVALID_ARGUMENT and "[1, n - 1]" in message
    with pytest.raises(hecuda.HeError, match=r"\[1, n - 1\]"):
        sp.OprfServer(sp.SymmetricPirConfig(bad.to_bytes(48, "big"))).computeResponses([query.tobytes()], SEED)


def test_null_pointers_negative_and_zero_count():
    key = np.frombuffer(KEY, dtype=np.uint8)
    query = np.frombuffer(O.blind(b"k", 3)[1], dtype=np.uint8)
    seed, out, status = np.zeros(32, dtype=np.uint8), np.zeros(145, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
    args = [P(key), P(query), 1, P(seed), P(out), P(status)]
    for i in (0, 1, 3, 4, 5):
        nulled = list(args)
        nulled[i] = None
        assert refusal(lambda lib: lib.hecuda_oprf_blind_evaluate(*nulled))[0] == ERR_INVALID_ARGUMENT
    negative = list(args)
    negative[2] = -1
    assert refusal(lambda lib: lib.hecuda_oprf_blind_evaluate(*negative))[0] == ERR_INVALID_ARGUMENT
    zero = list(args)
    zero[2] = 0
    assert refusal(lambda lib: lib.hecuda_oprf_blind_evaluate(*zero))[0] == 0
    assert sp.OprfServer(sp.SymmetricPirConfig(KEY)).computeResponses([], SEED) == []


def test_python_errors():
    with pytest.raises(pir.PirError, match="invalidOPRFKeySize"):
        sp.OprfServer(sp.SymmetricPirConfig(bytes(47)))
    config = sp.SymmetricPirConfig(KEY)
    config.oprfSecretKey = bytes(49)
    with pytest.raises(pir.PirError, match="invalidOPRFKeySize"):
        sp.OprfServer(config)
    server = sp.OprfServer(sp.SymmetricPirConfig(KEY))
    for query in invalid_queries() + [bytes(48)]:
        with pytest.raises(pir.PirError, match="invalidOprfQuery"):
            server.computeResponse(query, SEED)
    with pytest.raises(pir.PirError):
        server.computeResponses([], bytes(31))
