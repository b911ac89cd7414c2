"""Symmetric keyword PIR on the device: hecuda_oprf_evaluate, hecuda_oprf_public_key and hecuda_symmetric_pir_process
bit-exact against oracle/oprf_oracle.py and cryptography, a call past the 65535-row launch split, the reference's
roundTrip through keyword PIR, and the refusals."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda  # noqa: E402
from hecuda import keyword_pir as kw  # noqa: E402
from hecuda import pir  # noqa: E402
from hecuda import symmetric_pir as sp  # noqa: E402
from oracle import oprf_oracle as O  # noqa: E402
from oracle import oracle as orc  # noqa: E402

ERR_INVALID_ARGUMENT = -1
KEY = random.Random(20).randrange(1, O.N).to_bytes(48, "big")
TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)


def random_rows(seed, count):
    rng = random.Random(seed)
    lengths = [0, 1, 12, 111, 112, 127, 128, 300] + [rng.randrange(301) for _ in range(count - 8)]
    return [(rng.randbytes(n), rng.randbytes(rng.randrange(70))) for n in lengths[:count]]


@pytest.fixture(scope="module")
def rows():
    return random_rows(1, 2000)


@pytest.fixture(scope="module")
def expected(rows):
    return [O.evaluate(KEY, k) for k, _ in rows]


def test_oprf_evaluate_matches_the_restatement(rows, expected):
    out = sp.Oprf.evaluate(KEY, [k for k, _ in rows])
    assert out.shape == (len(rows), 48)
    assert [bytes(r) for r in out] == expected


def test_oprf_evaluate_long_input():
    data = random.Random(2).randbytes(65535)
    assert bytes(sp.Oprf.evaluate(KEY, [data])[0]) == O.evaluate(KEY, data)


@pytest.mark.parametrize("k", [1, 2, O.N - 1, O.N - 6, "key"])
def test_public_key_matches_cryptography(k):
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric import ec

    k = int.from_bytes(KEY, "big") if k == "key" else k
    expected = ec.derive_private_key(k, ec.SECP384R1()).public_key().public_bytes(
        serialization.Encoding.X962, serialization.PublicFormat.CompressedPoint)
    assert sp.Oprf.publicKey(k.to_bytes(48, "big")) == expected
    assert sp.SymmetricPirConfig(k.to_bytes(48, "big")).clientConfig().serverPublicKey == expected


def test_process_matches_the_restatement(rows, expected):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    out = kw.KeywordDatabase.symmetricPIRProcess(rows, sp.SymmetricPirConfig(KEY))
    for (keyword, value), h, (new_keyword, sealed) in zip(rows, expected, out):
        assert new_keyword == h[:16]
        assert sealed == O.seal(h, value)
        assert AESGCM(h[24:]).decrypt(h[:12], sealed, None) == value


def test_past_the_launch_split():
    """70000 rows in one call: rows on both sides of 65535 equal the restatement, and the call launches one more OPRF
    and one more seal kernel than a one-row call."""
    count = 70000
    rng = random.Random(3)
    keywords = [i.to_bytes(4, "little") + rng.randbytes(8) for i in range(count)]
    values = [rng.randbytes(i % 40) for i in range(count)]
    config = sp.SymmetricPirConfig(KEY)
    before = hecuda.kernel_launch_count()
    sp.symmetricPIRProcess([(keywords[0], values[0])], config)
    one = hecuda.kernel_launch_count() - before
    before = hecuda.kernel_launch_count()
    out = sp.symmetricPIRProcess(list(zip(keywords, values)), config)
    assert hecuda.kernel_launch_count() - before == one + 2 == 4
    before = hecuda.kernel_launch_count()
    hs = sp.Oprf.evaluate(KEY, keywords)
    assert hecuda.kernel_launch_count() - before == 2
    for i in (0, 65534, 65535, 65536, 69999):
        h = O.evaluate(KEY, keywords[i])
        assert bytes(hs[i]) == h
        assert out[i] == (h[:16], O.seal(h, values[i]))


def test_count_zero_launches_nothing():
    lib = hecuda.load_library()
    key = np.frombuffer(KEY, dtype=np.uint8)
    data = np.zeros(1, dtype=np.uint8)
    offsets = np.zeros(1, dtype=np.uint64)
    out = np.zeros(64, dtype=np.uint8)
    before = hecuda.kernel_launch_count()
    assert lib.hecuda_oprf_evaluate(hecuda._ptr(key), hecuda._ptr(data), hecuda._ptr(offsets), 0, hecuda._ptr(out)) == 0
    assert lib.hecuda_symmetric_pir_process(hecuda._ptr(key), hecuda._ptr(data), hecuda._ptr(offsets), hecuda._ptr(data),
                                            hecuda._ptr(offsets), 0, hecuda._ptr(out), hecuda._ptr(out)) == 0
    assert sp.symmetricPIRProcess([], sp.SymmetricPirConfig(KEY)) == []
    assert hecuda.kernel_launch_count() == before


def refusal(call):
    lib = hecuda.load_library()
    before = hecuda.kernel_launch_count()
    rc = call(lib)
    message = (lib.hecuda_last_error() or b"").decode()
    assert hecuda.kernel_launch_count() == before
    return rc, message


@pytest.mark.parametrize("bad", [0, O.N, O.N + 5, 2**384 - 1])
def test_bad_keys_are_refused(bad):
    key = np.frombuffer(bad.to_bytes(48, "big"), dtype=np.uint8)
    data, offsets = np.frombuffer(b"abc", dtype=np.uint8), np.array([0, 3], dtype=np.uint64)
    out = np.zeros(128, dtype=np.uint8)
    p = hecuda._ptr
    results = [
        refusal(lambda lib: lib.hecuda_oprf_public_key(p(key), p(out))),
        refusal(lambda lib: lib.hecuda_oprf_evaluate(p(key), p(data), p(offsets), 1, p(out))),
        refusal(lambda lib: lib.hecuda_symmetric_pir_process(p(key), p(data), p(offsets), p(data), p(offsets), 1, p(out),
                                                             p(out))),
    ]
    assert all(r == results[0] for r in results)
    assert results[0][0] == ERR_INVALID_ARGUMENT and "[1, n - 1]" in results[0][1]
    with pytest.raises(hecuda.HeError, match=r"\[1, n - 1\]"):
        sp.Oprf.evaluate(bad.to_bytes(48, "big"), [b"x"])


def test_bad_inputs_are_refused():
    p = hecuda._ptr
    key = np.frombuffer(KEY, dtype=np.uint8)
    long = np.zeros(65536, dtype=np.uint8)
    out = np.zeros(65536 + 64, dtype=np.uint8)
    too_long = np.array([0, 65536], dtype=np.uint64)
    decreasing = np.array([0, 5, 3], dtype=np.uint64)
    for offsets, count, needle in ((too_long, 1, "65535"), (decreasing, 2, "must not decrease")):
        zeros = np.zeros(count + 1, dtype=np.uint64)
        a = refusal(lambda lib: lib.hecuda_oprf_evaluate(p(key), p(long), p(offsets), count, p(out)))
        b = refusal(lambda lib: lib.hecuda_symmetric_pir_process(p(key), p(long), p(offsets), p(long), p(zeros), count,
                                                                 p(out), p(out)))
        assert a == b and a[0] == ERR_INVALID_ARGUMENT and needle in a[1]
    one, backwards = np.array([0, 1], dtype=np.uint64), np.array([4, 2], dtype=np.uint64)
    bad_values = refusal(lambda lib: lib.hecuda_symmetric_pir_process(p(key), p(long), p(one), p(long), p(backwards), 1,
                                                                      p(out), p(out)))
    assert bad_values[0] == ERR_INVALID_ARGUMENT and "value offsets must not decrease" in bad_values[1]
    negative = refusal(lambda lib: lib.hecuda_oprf_evaluate(p(key), p(long), p(too_long), -1, p(out)))
    assert negative[0] == ERR_INVALID_ARGUMENT
    with pytest.raises(pir.PirError, match="invalidOPRFKeySize"):
        sp.SymmetricPirConfig(bytes(47))
    with pytest.raises(pir.PirError, match="invalidOPRFKeySize"):
        sp.Oprf.evaluate(bytes(49), [b"x"])


@pytest.fixture(scope="module")
def test_context():
    n, t = 16, 1153
    ctx = hecuda.Context(n, orc.generate_primes(TEST_MODULI_BITS, False, n), t)
    yield ctx
    ctx.close()


def round_trip(g, database, encrypted, config):
    """SymmetricPirTests.roundTrip after processing: keyword PIR at the OPRF keyword, then the AES-GCM open."""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    keyword_config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(100), True, "noCompression",
                                         symmetricPirClientConfig=config.clientConfig())
    processed = kw.KeywordPirServer.processOnDevice(encrypted, keyword_config, g, symmetricPirConfig=config)
    assert processed.symmetricPirConfig is config
    server = kw.KeywordPirServer(g, processed)
    client = kw.KeywordPirClient(keyword_config.parameter, processed.pirParameter, g)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    indices = list(range(len(database)))
    random.Random(4).shuffle(indices)
    for index in indices[:10]:
        keyword, value = database[index]
        h = O.evaluate(config.oprfSecretKey, keyword)
        response = server.computeResponse(client.generateQuery(h[:16], sk), key)
        sealed = client.decrypt(response, h[:16], sk)
        assert sealed is not None
        assert AESGCM(h[24:]).decrypt(h[:12], sealed, None) == value
    key.close()
    processed.close()


def test_round_trip(test_context):
    g = test_context
    value_size = pir.bytesPerPlaintext(g) // 2
    rng = random.Random(5)
    database = [(b"keyword %d" % i, rng.randbytes(value_size)) for i in range(100)]
    config = sp.SymmetricPirConfig(KEY)
    assert config.clientConfig().serverPublicKey == O.public_key(KEY)
    round_trip(g, database, kw.KeywordDatabase.symmetricPIRProcess(database, config), config)


def test_round_trip_through_sharding(test_context):
    g = test_context
    value_size = pir.bytesPerPlaintext(g) // 2
    rng = random.Random(6)
    database = [(b"row %d" % i, rng.randbytes(value_size)) for i in range(200)]
    config = sp.SymmetricPirConfig(KEY)
    sharded = kw.KeywordDatabase(database, kw.Sharding.shardCount(2), symmetricPirConfig=config)
    assert sorted(sharded.shards) == ["0", "1"]
    expected = dict(O.symmetric_pir_process(KEY, database))
    assert sum(len(rows) for rows in sharded.shards.values()) == len(database)
    for rows in sharded.shards.values():
        assert all(expected[k] == v for k, v in rows)
    plain = dict(database)
    for shard_rows in sharded.shards.values():
        reverse = {O.evaluate(KEY, k)[:16]: (k, plain[k]) for k in plain}
        originals = [reverse[k] for k, _ in shard_rows]
        round_trip(g, originals, shard_rows, config)
    assert kw.KeywordDatabase(database, kw.Sharding.shardCount(2)).shards == \
        kw.KeywordDatabase(database, kw.Sharding.shardCount(2), symmetricPirConfig=None).shards
