"""The symmetric-PIR OPRF client on the device: hecuda_oprf_blind, hecuda_oprf_finalize, hecuda_symmetric_pir_open and
hecuda.symmetric_pir.OprfClient.  The OPRF property against hecuda_oprf_evaluate for 512 inputs, byte-equality with
oracle/oprf_oracle.py and tests/oprf_proof_ref.py on samples, every rejection inside a batch, a call past the
65535-query launch split, AES-GCM open against cryptography, the reference's oprfRoundtrip and roundTrip through the
device client alone, and the refusals."""
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
KEY = random.Random(70).randrange(1, O.N).to_bytes(48, "big")
OTHER_KEY = random.Random(71).randrange(1, O.N).to_bytes(48, "big")
SEED = bytes(range(32))
P = hecuda._ptr
N = O.N


def invalid_encodings():
    """Each kind of invalid element encoding: prefixes 0, 1 and 4, x = p, x > p, x off the curve, all zeros."""
    good = O.blind(b"neighbour", 5)[1]
    off_curve = next(x for x in range(1, 100) if not O.is_square((x ** 3 + O.A * x + O.B) % O.P))
    return [bytes([0]) + good[1:], bytes([1]) + good[1:], bytes([4]) + good[1:], b"\x02" + O.P.to_bytes(48, "big"),
            b"\x03" + (O.P + 1).to_bytes(48, "big"), b"\x02" + off_curve.to_bytes(48, "big"), bytes(49)]


def concatenate(blobs):
    offsets = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    return np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8), offsets


def packed(blobs):
    """The blobs back to back.  Keep the array in a variable while the library reads its pointer."""
    return np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)


def blind(inputs, blinds):
    lib = hecuda.load_library()
    data, offsets = concatenate(inputs)
    count = len(inputs)
    queries = np.full((max(count, 1), 49), 7, dtype=np.uint8)
    status = np.full(max(count, 1), 7, dtype=np.uint8)
    scalars = packed([r.to_bytes(48, "big") for r in blinds])
    rc = lib.hecuda_oprf_blind(P(data), P(offsets), count, P(scalars), P(queries), P(status))
    assert rc == 0, (lib.hecuda_last_error() or b"").decode()
    return [q.tobytes() for q in queries[:count]], status[:count].tolist()


def finalize(inputs, blinds, queries, responses, key=KEY):
    lib = hecuda.load_library()
    data, offsets = concatenate(inputs)
    count = len(inputs)
    outputs = np.full((max(count, 1), 48), 7, dtype=np.uint8)
    status = np.full(max(count, 1), 7, dtype=np.uint8)
    pk = np.frombuffer(O.public_key(key), dtype=np.uint8)
    scalars, elements, answers = packed([r.to_bytes(48, "big") for r in blinds]), packed(queries), packed(responses)
    rc = lib.hecuda_oprf_finalize(P(pk), P(data), P(offsets), count, P(scalars), P(elements), P(answers), P(outputs),
                                  P(status))
    assert rc == 0, (lib.hecuda_last_error() or b"").decode()
    return [o.tobytes() for o in outputs[:count]], status[:count].tolist()


def open_entries(outputs, entries):
    lib = hecuda.load_library()
    sealed, offsets = concatenate(entries)
    count = len(entries)
    values = np.full(max(int(offsets[-1]), 1), 7, dtype=np.uint8)
    status = np.full(max(count, 1), 7, dtype=np.uint8)
    hashes = packed(outputs)
    rc = lib.hecuda_symmetric_pir_open(P(hashes), P(sealed), P(offsets), count, P(values), P(status))
    assert rc == 0, (lib.hecuda_last_error() or b"").decode()
    raw = values.tobytes()
    return [raw[int(offsets[i]):int(offsets[i + 1])] for i in range(count)], status[:count].tolist()


def respond(queries, key=KEY):
    responses = sp.OprfServer(sp.SymmetricPirConfig(key)).computeResponses(queries, SEED)
    assert all(r is not None for r in responses)
    return responses


@pytest.fixture(scope="module")
def batch():
    rng = random.Random(72)
    inputs = [rng.randbytes(rng.randrange(0, 65)) for _ in range(511)] + [rng.randbytes(65535)]
    blinds = [rng.randrange(1, N) for _ in inputs]
    queries, status = blind(inputs, blinds)
    assert status == [0] * len(inputs)
    responses = respond(queries)
    return inputs, blinds, queries, responses


def test_oprf_property(batch):
    """blind -> OprfServer -> finalize equals Oprf.evaluate for 512 inputs of 0 to 64 bytes and one of 65535; sampled
    queries equal the oracle's Blind and sampled outputs the restatement's verifying Finalize."""
    inputs, blinds, queries, responses = batch
    outputs, status = finalize(inputs, blinds, queries, responses)
    assert status == [0] * len(inputs)
    assert outputs == [bytes(h) for h in sp.Oprf.evaluate(KEY, inputs)]
    pk = O.public_key(KEY)
    for i in (0, 1, 255, 511):
        assert queries[i] == O.blind(inputs[i], blinds[i])[1]
    for i in (0, 511):
        assert outputs[i] == R.finalize_verifiable(inputs[i], blinds[i], responses[i], pk)


def test_oracle_made_responses(batch):
    """Responses built by the restatement's BlindEvaluate finalize to the same outputs as the device server's."""
    inputs, blinds, queries, responses = batch
    picks = [0, 3, 100, 510]
    made = [R.blind_evaluate_verifiable(KEY, queries[i], b"\x05" * 32) for i in picks]
    outputs, status = finalize([inputs[i] for i in picks], [blinds[i] for i in picks], [queries[i] for i in picks], made)
    assert status == [0] * len(picks)
    assert outputs == [O.evaluate(KEY, inputs[i]) for i in picks]


def flip(b: bytes, byte: int, bit: int = 0) -> bytes:
    return b[:byte] + bytes([b[byte] ^ (1 << bit)]) + b[byte + 1:]


def decodes(e: bytes) -> bool:
    try:
        O.deserialize_element(e)
        return True
    except ValueError:
        return False


def test_rejections_inside_a_batch(batch):
    """Each tampering gets its status and 48 zero bytes; the queries around it equal a batch without it."""
    inputs, blinds, queries, responses = [x[:40] for x in batch]
    other = respond(queries[:1], OTHER_KEY)[0]
    r0 = responses[0]
    flipped_d = next(f for f in (flip(r0, 48, b) for b in range(8)) if decodes(f[:49]))
    bad = [  # (blind, query, response, status) for input 0
        (blinds[0], queries[0], flipped_d, 1),
        (blinds[0], queries[0], flip(r0, 60), 1),
        (blinds[0], queries[0], flip(r0, 120), 1),
        (blinds[0], queries[0], r0[:49] + N.to_bytes(48, "big") + r0[97:], 1),
        (blinds[0], queries[0], r0[:97] + N.to_bytes(48, "big"), 1),
        (blinds[0], queries[0], other, 1),              # a response under a different key
        (blinds[0], queries[0], responses[1], 1),       # swapped responses
        (blinds[0], queries[1], r0, 1),                 # the query another response answers
    ] + [(blinds[0], queries[0], e + r0[49:], 1) for e in invalid_encodings()] + \
        [(blinds[0], e, r0, 2) for e in invalid_encodings()] + \
        [(r, queries[0], r0, 2) for r in (0, N, 2**384 - 1)]
    mixed = list(zip(inputs, blinds, queries, responses))
    where = []
    for j, (r, q, resp, _) in enumerate(bad):
        at = 2 + 2 * j
        mixed.insert(at, (inputs[0], r, q, resp))
        where.append(at)
    outputs, status = finalize(*[list(x) for x in zip(*mixed)])
    assert [status[i] for i in where] == [s for *_, s in bad]
    assert all(outputs[i] == bytes(48) for i in where)
    clean, clean_status = finalize(inputs, blinds, queries, responses)
    assert clean_status == [0] * len(inputs)
    assert [o for i, o in enumerate(outputs) if i not in where] == clean
    assert [s for i, s in enumerate(status) if i not in where] == clean_status


def test_invalid_blinds_when_blinding():
    queries, status = blind([b"a", b"b", b"c", b"d"], [5, 0, N, 2**384 - 1])
    assert status == [0, 1, 1, 1]
    assert queries[0] == O.blind(b"a", 5)[1] and queries[1:] == [bytes(49)] * 3


def test_past_the_launch_split():
    """70000 queries in one call equal the calls on [0, 65535) and [65535, 70000), and each call launches one more
    kernel of each per-query kind than a one-query call."""
    count = 70000
    inputs = [b"split %d" % (i % 97) for i in range(count)]
    blinds = [1000 + 7 * i for i in range(count)]
    before = hecuda.kernel_launch_count()
    blind(inputs[:1], blinds[:1])
    assert hecuda.kernel_launch_count() - before == 1
    before = hecuda.kernel_launch_count()
    queries, status = blind(inputs, blinds)
    assert hecuda.kernel_launch_count() - before == 2
    assert status == [0] * count
    assert blind(inputs[:65535], blinds[:65535])[0] + blind(inputs[65535:], blinds[65535:])[0] == queries
    responses = respond(queries)
    before = hecuda.kernel_launch_count()
    finalize(inputs[:1], blinds[:1], queries[:1], responses[:1])
    assert hecuda.kernel_launch_count() - before == 2
    before = hecuda.kernel_launch_count()
    outputs, status = finalize(inputs, blinds, queries, responses)
    assert hecuda.kernel_launch_count() - before == 4
    assert status == [0] * count
    first = finalize(inputs[:65535], blinds[:65535], queries[:65535], responses[:65535])[0]
    second = finalize(inputs[65535:], blinds[65535:], queries[65535:], responses[65535:])[0]
    assert first + second == outputs
    expected = {bytes(m): bytes(h) for m, h in zip(inputs[:97], sp.Oprf.evaluate(KEY, inputs[:97]))}
    assert all(outputs[i] == expected[inputs[i]] for i in (0, 65534, 65535, 65536, 69999))
    for i in (65535, 69999):
        assert queries[i] == O.blind(inputs[i], blinds[i])[1]


LENGTHS = (0, 1, 15, 16, 17, 4096)


@pytest.fixture(scope="module")
def sealed_rows():
    rng = random.Random(73)
    rows = [(b"row %d" % i, rng.randbytes(n)) for i, n in enumerate(LENGTHS)]
    processed = sp.symmetricPIRProcess(rows, sp.SymmetricPirConfig(KEY))
    outputs = [bytes(h) for h in sp.Oprf.evaluate(KEY, [k for k, _ in rows])]
    return rows, processed, outputs


def test_open_matches_aesgcm(sealed_rows):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM

    rows, processed, outputs = sealed_rows
    values, status = open_entries(outputs, [v for _, v in processed])
    assert status == [0] * len(rows)
    for (_, value), (_, sealed), h, got in zip(rows, processed, outputs, values):
        assert AESGCM(h[24:48]).decrypt(h[:12], sealed, None) == value
        assert got == value + bytes(16)


def test_open_rejects_inside_a_batch(sealed_rows):
    """A tampered tag, a tampered ciphertext, a wrong OPRF output and entries shorter than a tag get status 1 and a
    zeroed slot; the entries around them open as in a clean batch."""
    rows, processed, outputs = sealed_rows
    entries = [v for _, v in processed]
    bad = [(outputs[5], flip(entries[5], len(entries[5]) - 1)), (outputs[5], flip(entries[5], 100, 2)),
           (outputs[4], entries[5]), (outputs[0], entries[0][:15]), (outputs[0], b"")]
    mixed = list(zip(outputs, entries))
    where = []
    for j, item in enumerate(bad):
        mixed.insert(1 + 2 * j, item)
        where.append(1 + 2 * j)
    values, status = open_entries([h for h, _ in mixed], [e for _, e in mixed])
    assert [status[i] for i in where] == [1] * len(bad)
    assert all(values[i] == bytes(len(mixed[i][1])) for i in where)
    assert [v for i, v in enumerate(values) if i not in where] == [value + bytes(16) for _, value in rows]
    client = sp.OprfClient(sp.SymmetricPirConfig(KEY).clientConfig())
    parsed = [sp.ParsedOprfOutput.fromOprfOutput(h, client.configType) for h, _ in mixed]
    opened = client.decryptMany([e for _, e in mixed], parsed)
    assert [o for i, o in enumerate(opened) if i in where] == [None] * len(bad)
    assert [o for i, o in enumerate(opened) if i not in where] == [value for _, value in rows]
    with pytest.raises(pir.PirError, match="authenticationFailure"):
        client.decrypt(mixed[where[0]][1], parsed[where[0]])


def test_oprf_roundtrip():
    """SymmetricPIRTests.oprfRoundtrip through the device client: one keyword twice gives different queries and equal
    outputs."""
    config = sp.SymmetricPirConfig(KEY)
    server = sp.OprfServer(config)
    client = sp.OprfClient(config.clientConfig())
    keyword = bytes([1, 2, 3, 4, 5])
    outputs, queries = [], []
    for _ in range(2):
        context = client.queryContext(keyword)
        queries.append(context.query)
        outputs.append(client.parse(server.computeResponse(context.query), context))
    assert queries[0] != queries[1]
    assert outputs[0] == outputs[1]
    h = O.evaluate(KEY, keyword)
    assert outputs[0] == sp.ParsedOprfOutput(h[:16], h[:12], h[24:])
    assert "****" in repr(outputs[0]) and h[24:].hex() not in repr(outputs[0])
    context = client.queryContexts([keyword], [12345])[0]
    assert context.query == O.blind(keyword, 12345)[1] and "12345" not in repr(context)


@pytest.fixture(scope="module")
def test_context():
    import oracle.oracle as orc

    n, t = 16, 1153
    ctx = hecuda.Context(n, orc.generate_primes([55, 52, 62, 58], False, n), t)
    yield ctx
    ctx.close()


def round_trip(g, database, encrypted, config):
    """SymmetricPirTests.roundTrip (_TestUtilities/PirUtilities/SymmetricPirTests.swift:33-95) with the device OPRF
    client: OPRF through OprfServer, keyword PIR at the oblivious keyword, then the AES-GCM open."""
    keyword_config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(100), True, "noCompression",
                                         symmetricPirClientConfig=config.clientConfig())
    processed = kw.KeywordPirServer.processOnDevice(encrypted, keyword_config, g, symmetricPirConfig=config)
    server = kw.KeywordPirServer(g, processed)
    client = kw.KeywordPirClient(keyword_config.parameter, processed.pirParameter, g)
    oprf_server = sp.OprfServer(config)
    oprf_client = sp.OprfClient(keyword_config.symmetricPirClientConfig)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    indices = list(range(len(database)))
    random.Random(74).shuffle(indices)
    picked = [database[i] for i in indices[:10]]
    contexts = oprf_client.queryContexts([k for k, _ in picked])
    parsed = oprf_client.parseMany(oprf_server.computeResponses([c.query for c in contexts]), contexts)
    sealed = []
    for p in parsed:
        response = server.computeResponse(client.generateQuery(p.obliviousKeyword, sk), key)
        sealed.append(client.decrypt(response, p.obliviousKeyword, sk))
        assert sealed[-1] is not None
    assert oprf_client.decryptMany(sealed, parsed) == [v for _, v in picked]
    assert oprf_client.decrypt(sealed[0], parsed[0]) == picked[0][1]
    key.close()
    processed.close()


def test_round_trip(test_context):
    g = test_context
    rng = random.Random(75)
    database = [(b"keyword %d" % i, rng.randbytes(pir.bytesPerPlaintext(g) // 2)) for i in range(100)]
    config = sp.SymmetricPirConfig(KEY)
    round_trip(g, database, kw.KeywordDatabase.symmetricPIRProcess(database, config), config)


def test_round_trip_through_sharding(test_context):
    g = test_context
    rng = random.Random(76)
    database = [(b"row %d" % i, rng.randbytes(pir.bytesPerPlaintext(g) // 2)) for i in range(200)]
    config = sp.SymmetricPirConfig(KEY)
    sharded = kw.KeywordDatabase(database, kw.Sharding.shardCount(2), symmetricPirConfig=config)
    plain = dict(database)
    reverse = {bytes(h)[:16]: (k, plain[k]) for k, h in zip(plain, sp.Oprf.evaluate(KEY, list(plain)))}
    assert len(sharded.shards) == 2
    for shard_rows in sharded.shards.values():
        round_trip(g, [reverse[k] for k, _ in shard_rows], shard_rows, config)


def refusal(call):
    lib = hecuda.load_library()
    before = hecuda.kernel_launch_count()
    rc = call(lib)
    message = (lib.hecuda_last_error() or b"").decode()
    assert hecuda.kernel_launch_count() == before
    return rc, message


def test_refusals():
    """Null pointers, a negative count, decreasing offsets, an input over 65535 bytes and an invalid public key are
    refused with no kernel launched; a count of 0 succeeds."""
    data, offsets = concatenate([b"ab", b"c"])
    blinds = packed([(5).to_bytes(48, "big")] * 2)
    q = np.zeros((2, 49), dtype=np.uint8)
    resp, out, status = np.zeros((2, 145), dtype=np.uint8), np.zeros((2, 48), dtype=np.uint8), np.zeros(2, dtype=np.uint8)
    pk = np.frombuffer(O.public_key(KEY), dtype=np.uint8)
    decreasing = np.array([0, 2, 1], dtype=np.uint64)
    long_input = np.zeros(65536, dtype=np.uint8)
    too_long = np.array([0, 65536], dtype=np.uint64)
    calls = {
        "hecuda_oprf_blind": [P(data), P(offsets), 2, P(blinds), P(q), P(status)],
        "hecuda_oprf_finalize": [P(pk), P(data), P(offsets), 2, P(blinds), P(q), P(resp), P(out), P(status)],
    }
    for name, args in calls.items():
        count_at = args.index(2)
        for i in range(len(args)):
            if i == count_at:
                continue
            nulled = list(args)
            nulled[i] = None
            assert refusal(lambda lib: getattr(lib, name)(*nulled))[0] == ERR_INVALID_ARGUMENT, (name, i)
        for count, offs, inp in ((-1, offsets, data), (2, decreasing, data), (1, too_long, long_input)):
            changed = list(args)
            changed[count_at], changed[count_at - 1], changed[count_at - 2] = count, P(offs), P(inp)
            assert refusal(lambda lib: getattr(lib, name)(*changed))[0] == ERR_INVALID_ARGUMENT, (name, count)
        zero = list(args)
        zero[count_at] = 0
        assert refusal(lambda lib: getattr(lib, name)(*zero))[0] == 0
    for bad_pk in invalid_encodings():
        key = np.frombuffer(bad_pk, dtype=np.uint8)
        for count in (2, 0):
            rc, message = refusal(lambda lib: lib.hecuda_oprf_finalize(P(key), P(data), P(offsets), count, P(blinds),
                                                                        P(q), P(resp), P(out), P(status)))
            assert rc == ERR_INVALID_ARGUMENT and "public key" in message
    sealed_args = [P(out), P(data), P(offsets), 2, P(data), P(status)]
    for i in (0, 1, 2, 4, 5):
        nulled = list(sealed_args)
        nulled[i] = None
        assert refusal(lambda lib: lib.hecuda_symmetric_pir_open(*nulled))[0] == ERR_INVALID_ARGUMENT
    for count, offs in ((-1, offsets), (2, decreasing)):
        changed = list(sealed_args)
        changed[3], changed[2] = count, P(offs)
        assert refusal(lambda lib: lib.hecuda_symmetric_pir_open(*changed))[0] == ERR_INVALID_ARGUMENT
    zero = list(sealed_args)
    zero[3] = 0
    assert refusal(lambda lib: lib.hecuda_symmetric_pir_open(*zero))[0] == 0


def test_python_errors():
    config = sp.SymmetricPirConfig(KEY)
    for bad_pk in invalid_encodings() + [bytes(48)]:
        with pytest.raises(pir.PirError, match="invalid OPRF public key"):
            sp.OprfClient(sp.SymmetricPirClientConfig(bad_pk))
    client = sp.OprfClient(config.clientConfig())
    server = sp.OprfServer(config)
    context = client.queryContext(b"word")
    response = server.computeResponse(context.query)
    other = sp.OprfServer(sp.SymmetricPirConfig(OTHER_KEY)).computeResponse(context.query)
    with pytest.raises(pir.PirError, match="invalidOprfResponse"):
        client.parse(other, context)
    assert client.parseMany([response, other, response[:100]], [context] * 3)[1:] == [None, None]
    assert client.parseMany([response], [context])[0] == client.parse(response, context)
    for blinds in ([0], [N], [2**384]):
        with pytest.raises(pir.PirError, match="invalid OPRF blind"):
            client.queryContexts([b"x"], blinds)
    assert client.queryContexts([]) == [] and client.parseMany([], []) == [] and client.decryptMany([], []) == []
