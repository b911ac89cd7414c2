"""PIR in the reference's protobuf messages on the GPU: EncryptedIndices and SerializedEvaluationKey in, PIRResponse out
(hecuda_mulpir_compute_response_clients_proto, hecuda_evk_create_proto_many, hecuda_pir_request_fields_read).

- Parity: every client's PIRResponse is byte-identical to the restatement's framing (tests/pir_proto_ref.py) around the
  _clients_wire reply of the same poly0 and seeds, at the C4 shape and at a two-chunk, two-dimension shape, for 1, 2,
  16 and 17 clients (across a group boundary).
- Keys: fromProtoMany gives the words of fromSerializedMany for the same payloads, whatever the map order.
- .full query ciphertexts answer like their seeded form.
- End to end: device MulPir and keyword-PIR clients put a key and a query in a PIRRequest, the server answers from the
  request's ranges, and every client of a batch of 16 decrypts its entry.
- Errors: a bad client is named and leaves `out` untouched; keys with different Galois sets are refused."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
import pir_proto_ref as ref
from hecuda import keyword_pir as kw
from hecuda import pir
from rlwe_shapes import read_device

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:357-367)
N, T = 4096, 17
ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = -1, -2


@pytest.fixture(scope="module")
def g():
    ctx = hecuda.Context(N, PIR_MODULI, T)
    yield ctx
    ctx.close()


def query_sizes(g):
    return ref.poly_sizes(N, [q.bit_length() for q in g.coefficientModuli[:g.L]])


def reply_sizes(g):
    return ref.poly_sizes(N, [g.coefficientModuli[0].bit_length()])


def random_server(g, entries, entry_size, seed):
    """A MulPir server over random plaintext rows (byte parity needs no real entries)."""
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(entries, entry_size, 2, 1, True, "hybridCompression", False), g)
    chunks = -(-param.encodedEntrySize // pir.bytesPerPlaintext(g))
    rows = np.random.default_rng(seed).integers(0, T, size=(chunks * int(np.prod(param.dimensions)), N), dtype=np.uint64)
    return pir.MulPirServer(param, g, [pir.ProcessedDatabase(g, rows, None, evalFormat=False)])


def clients(g, server, count, seed):
    """count device clients: (secret key, key message, key form, query message, indices)."""
    client = pir.MulPirClient(server.parameter, g)
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        sk = hecuda.SecretKey.generate(g)
        key, form = hecuda.EvaluationKey.generate(g, client.evaluationKeyConfig, sk, wire=True)
        key.close()
        indices = [rng.randrange(server.parameter.entryCount)]
        out.append(dict(sk=sk, form=form, key_message=pir.evaluationKeyMessage(g, form),
                        query=client.queryMessage(indices, sk), indices=indices))
    return client, out


def framed_wire_replies(g, server, cs, keys, indices_count=1):
    """The restatement's PIRResponse around each client's _clients_wire reply of the same poly0 and seeds."""
    sz = query_sizes(g)
    cts = [ref.parse_encrypted_indices(c["query"], sz)[0] for c in cs]
    poly0 = np.stack([np.frombuffer(b"".join(ct[1] for ct in q), np.uint8) for q in cts])
    seeds = np.stack([np.frombuffer(b"".join(ct[2] for ct in q), np.uint8) for q in cts])
    replies, skips = pir.PirWire.computeResponses(server, poly0.reshape(len(cs), len(cts[0]), -1),
                                                  seeds.reshape(len(cs), len(cts[0]), 32), keys, indices_count)
    half = reply_sizes(g)(skips[0])
    return [ref.encode_pir_response([[(r[:half].tobytes(), r[half:].tobytes()) for r in reply] for reply in client_replies],
                                    skips) for client_replies in replies]


SHAPES = {"c4": (1 << 20, 64), "two_chunks": (3000, 3000)}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_parity_with_the_wire_path(g, shape):
    entries, entry_size = SHAPES[shape]
    server = random_server(g, entries, entry_size, seed=entries)
    if shape == "two_chunks":
        assert server.chunkCount == 2 and len(server.parameter.dimensions) == 2
    _, cs = clients(g, server, 17, seed=entry_size)
    keys = hecuda.EvaluationKey.fromProtoMany(g, [c["key_message"] for c in cs])
    for count in (1, 2, 16, 17):
        got = pir.PirWire.computeResponsesProto(server, [c["query"] for c in cs[:count]], keys[:count])
        want = framed_wire_replies(g, server, cs[:count], keys[:count])
        assert len(got) == count
        for j in range(count):
            assert got[j] == want[j], (count, j)
    size = C.c_uint64()
    skips = pir.skipLSBsForDecryption(g)
    assert hecuda.load_library().hecuda_mulpir_response_proto_byte_count(g._h, server.chunkCount, 1, skips[0], skips[1],
                                                                         C.byref(size)) == 0
    assert size.value == len(got[0])
    for k in keys:
        k.close()


def test_keys_equal_serialized_many_in_any_map_order(g):
    server = random_server(g, 3000, 3000, seed=1)
    _, cs = clients(g, server, 3, seed=2)
    forms = [c["form"] for c in cs]
    shuffled = []
    for j, f in enumerate(forms):
        items = list(f["galois"].items())
        random.Random(j).shuffle(items)
        shuffled.append(pir.evaluationKeyMessage(g, dict(f, galois=dict(items))))
    # a shuffled message parses to the same keys in the restatement, and in the library to the same words
    sz = ref.poly_sizes(N, [q.bit_length() for q in g.coefficientModuli])
    assert ref.parse_evaluation_key(shuffled[1], sz, g.L)[0] == \
        dict(sorted(ref.parse_evaluation_key(cs[1]["key_message"], sz, g.L)[0].items()))
    got = hecuda.EvaluationKey.fromProtoMany(g, shuffled)
    want = hecuda.EvaluationKey.fromSerializedMany(g, forms)
    for a, b in zip(got, want):
        assert np.array_equal(read_device(*a.deviceBuffer()), read_device(*b.deviceBuffer()))
        for e in b.galoisElements:
            assert np.array_equal(read_device(*a.galoisDeviceBuffer(e)), read_device(*b.galoisDeviceBuffer(e)))
    for k in got + want:
        k.close()


def test_full_query_ciphertexts_answer_like_seeded(g):
    server = random_server(g, 3000, 3000, seed=3)
    _, cs = clients(g, server, 2, seed=4)
    keys = hecuda.EvaluationKey.fromProtoMany(g, [c["key_message"] for c in cs])
    sz = query_sizes(g)
    full = []
    for c in cs:
        cts, calls = ref.parse_encrypted_indices(c["query"], sz)
        poly0 = np.stack([np.frombuffer(ct[1], np.uint8) for ct in cts])
        seeds = np.stack([np.frombuffer(ct[2], np.uint8) for ct in cts])
        expanded = hecuda.Bfv.expandSeeded(g, poly0, seeds)  # (count, 2, L, N)
        polys = hecuda.Bfv.serialize(g, expanded)  # (count x 2, bytes)
        # client 0 writes skip_lsbs [0, 0], client 1 leaves them out (both mean no dropped bits)
        skips = [0, 0] if not full else []
        full.append(ref.encode_encrypted_indices(
            [("full", ref.full_polys(polys[2 * i].tobytes(), polys[2 * i + 1].tobytes()), skips, 1) for i in range(len(cts))],
            calls))
    seeded = pir.PirWire.computeResponsesProto(server, [c["query"] for c in cs], keys)
    assert pir.PirWire.computeResponsesProto(server, full, keys) == seeded
    mixed = [full[0], cs[1]["query"]]
    assert pir.PirWire.computeResponsesProto(server, mixed, keys) == seeded
    for k in keys:
        k.close()


def request_round_trip(g, server_call, requests):
    """The server side of a batch of PIRRequests: the ranges from PirRequest.fields into the key and response calls."""
    fields = [pir.PirRequest.fields(r) for r in requests]
    key_messages = [r[f["evaluationKey"][0]:sum(f["evaluationKey"])] for r, f in zip(requests, fields)]
    queries = [r[f["query"][0]:sum(f["query"])] for r, f in zip(requests, fields)]
    keys = hecuda.EvaluationKey.fromProtoMany(g, key_messages)
    responses = server_call(queries, keys)
    for k in keys:
        k.close()
    return fields, responses


def test_mulpir_end_to_end(g):
    rng = random.Random(5)
    entries = [bytes(rng.randrange(256) for _ in range(100)) for _ in range(2000)]
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(len(entries), 100, 2, 1, True, "hybridCompression", False), g)
    server = pir.MulPirServer(param, g, [pir.MulPirServer.processOnDevice(entries, g, param)])
    client = pir.MulPirClient(param, g)
    batch = []
    for j in range(16):
        sk = hecuda.SecretKey.generate(g)
        key, key_message = client.evaluationKeyMessage(sk)
        key.close()
        indices = [rng.randrange(len(entries))]
        request = ref.encode_pir_request(shard_index=j % 3, query=client.queryMessage(indices, sk), shard_id=f"shard{j}",
                                         configuration_hash=b"\x01\x02", evaluation_key=key_message,
                                         key_metadata=(1000 + j, b"id%d" % j))
        batch.append((sk, indices, request))
    fields, responses = request_round_trip(
        g, lambda q, k: pir.PirWire.computeResponsesProto(server, q, k), [r for _, _, r in batch])
    for j, ((sk, indices, request), f, response) in enumerate(zip(batch, fields, responses)):
        assert f == ref.parse_pir_request(request)
        assert (f["shardIndex"], f["shardId"], f["keyTimestamp"], f["keyIdentifier"]) == (j % 3, f"shard{j}", 1000 + j,
                                                                                            b"id%d" % j)
        assert client.decryptResponseMessage(response, indices, sk) == [entries[i] for i in indices], j


def test_keyword_pir_end_to_end(g):
    rng = random.Random(6)
    rows = [(b"key%d" % i, bytes(rng.randrange(256) for _ in range(20))) for i in range(300)]
    config = kw.KeywordPirConfig(2, kw.CuckooTableConfig(2, 100, 100, kw.AllowExpansion(1.1, 0.9)), False, "noCompression")
    processed = kw.KeywordPirServer.processOnDevice(rows, config, g, kw.Rng.counter(3))
    server = kw.KeywordPirServer(g, processed)
    assert server.hashFunctionCount > 1
    client = kw.KeywordPirClient(processed.keywordPirParameter, processed.pirParameter, g)
    batch = []
    for j in range(16):
        sk = hecuda.SecretKey.generate(g)
        key, key_message = client.evaluationKeyMessage(sk)
        key.close()
        keyword, value = rows[rng.randrange(len(rows))]
        request = ref.encode_pir_request(query=client.queryMessage(keyword, sk), evaluation_key=key_message,
                                         metadata=(7, b"k"))
        batch.append((sk, keyword, value, request))
    _, responses = request_round_trip(g, server.computeResponsesProto, [r for *_, r in batch])
    for j, ((sk, keyword, value, _), response) in enumerate(zip(batch, responses)):
        assert client.decryptResponseMessage(response, keyword, sk) == value, j


def raw_call(g, server, messages, keys, indices_count=1):
    """hecuda_mulpir_compute_response_clients_proto into a filled buffer: (rc, error, buffer unchanged)."""
    lib = hecuda.load_library()
    out = np.full(1 << 20, 0xAB, dtype=np.uint8)
    bufs = [np.frombuffer(m, np.uint8) if m else np.zeros(1, np.uint8) for m in messages]
    counts = np.array([len(m) for m in messages], dtype=np.uint64)
    dims = (C.c_int32 * len(server.parameter.dimensions))(*server.parameter.dimensions)
    dbs = (C.c_void_p * 1)(server.databases[0]._h)
    skips = pir.skipLSBsForDecryption(g)
    rc = lib.hecuda_mulpir_compute_response_clients_proto(
        g._h, (C.c_void_p * len(keys))(*[k._h for k in keys]), len(keys), dbs, 1, dims, len(dims), server.chunkCount,
        (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs]), counts.ctypes.data_as(C.c_void_p), indices_count,
        skips[0], skips[1], out.ctypes.data_as(C.c_void_p))
    return rc, lib.hecuda_last_error().decode() if rc else "", bool((out == 0xAB).all())


def test_errors(g):
    server = random_server(g, 3000, 3000, seed=7)
    _, cs = clients(g, server, 3, seed=8)
    keys = hecuda.EvaluationKey.fromProtoMany(g, [c["key_message"] for c in cs])
    good = [c["query"] for c in cs]
    sz = query_sizes(g)
    cts, calls = ref.parse_encrypted_indices(good[1], sz)
    bad = {
        "num_pir_calls": ref.encode_encrypted_indices(cts, 2),
        "ciphertext_count": ref.encode_encrypted_indices(cts + cts, calls),
        "short_seed": ref.encode_encrypted_indices([("seeded", cts[0][1], cts[0][2][:31])] + cts[1:], calls),
        "truncated": good[1][:-1],
        "correction": ref.encode_encrypted_indices([("full", ref.full_polys(cts[0][1], cts[0][1]), [0, 0], 2)] + cts[1:],
                                                   calls),
    }
    for name, message in bad.items():
        rc, err, untouched = raw_call(g, server, [good[0], message, good[2]], keys)
        assert rc == (ERR_UNSUPPORTED if name == "correction" else ERR_INVALID_ARGUMENT), name
        assert err.startswith("client 1: "), (name, err)
        assert untouched, name
    assert raw_call(g, server, good, keys)[0] == 0
    # keys whose Galois sets differ
    other = dict(cs[1]["form"])
    other["galois"] = dict(list(other["galois"].items())[:-1])
    with pytest.raises(hecuda.HeError, match="client 1: Galois elements differ"):
        hecuda.EvaluationKey.fromProtoMany(g, [cs[0]["key_message"], pir.evaluationKeyMessage(g, other)])
    # a repeated element, and a relinearization key present for one client only
    sizes = ref.poly_sizes(N, [q.bit_length() for q in g.coefficientModuli])
    galois, relin = ref.parse_evaluation_key(cs[0]["key_message"], sizes, g.L)
    e0 = next(iter(galois))
    with pytest.raises(hecuda.HeError, match="client 0: repeated Galois element"):
        hecuda.EvaluationKey.fromProtoMany(g, [ref.encode_evaluation_key([(e0, galois[e0]), (e0, galois[e0])], relin)])
    if relin is not None:
        with pytest.raises(hecuda.HeError, match="client 1: relinearization key absent"):
            hecuda.EvaluationKey.fromProtoMany(g, [cs[0]["key_message"], ref.encode_evaluation_key(list(galois.items()))])
    for k in keys:
        k.close()
