"""SimplePIR in the reference's protobuf messages on the GPU (hecuda_simple_pir_compute_response_proto): every response
equals the restatement's framing (tests/simple_pir_proto_ref.py) of the words hecuda_simple_pir_compute_response gives
for the message's rows, over ragged 32- and 64-bit shards, ct 28 to 61, 1 to 64 messages with random row counts,
empty requests, a request past 2^20 varints and 33 shards; unpacked and split-packed data answer like packed data;
every refusal names its message and leaves the output untouched; the tool's files round-trip through the config; the
launch count does not depend on the message count; and nothing is leaked."""
import ctypes as C
import gc
import os

import numpy as np
import pytest

import hecuda
import simple_pir_proto_ref as ref
from hecuda import simple_pir as sp

pytestmark = pytest.mark.gpu


def enc(pt=14, ct=42, n=16, std=3.2):
    return sp.SimplePirEncryptionParams(pt, ct, n, std, "unchecked")


def _free_device_bytes():
    import torch

    torch.cuda.synchronize()
    cuda = C.CDLL("libcuda.so.1")
    dev, pool = C.c_int(), C.c_void_p()
    assert cuda.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
    assert cuda.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cuda.cuMemPoolTrimTo(pool, C.c_size_t(0)) == 0
    return torch.cuda.mem_get_info()[0]


@pytest.fixture(scope="module", autouse=True)
def no_device_leak():
    before = _free_device_bytes()
    yield
    gc.collect()
    leaked = before - _free_device_bytes()
    assert leaked < 64 << 20, f"the module leaves {leaked / 2**20:.1f} MiB of device memory allocated"


def ragged_server(rng, shapes, scalar, ct=42, pt=14):
    """shapes: (entry bytes, entriesPerColumn, chunksPerEntry, databaseColumns) per shard, random DB' values."""
    dbs, hints, params = [], [], []
    for size, epc, cpe, k in shapes:
        prm = sp.SimplePirParameters(enc(pt, ct), size, epc, cpe, k)
        db = rng.integers(0, 1 << pt, size=(prm.columnSize, k), dtype=np.uint64).astype(scalar)
        dbs.append(sp.SimplePirDatabase.create(db, prm, scalar))
        hints.append(np.zeros((prm.columnSize, 16), scalar))
        params.append(prm)
    return sp.SimplePirShardedServer(dbs, hints, params, scalar)


def expected_words(server, shard, rows):
    """hecuda_simple_pir_compute_response's words for `rows` (R x K_s): padded to whole requests, extra rows dropped."""
    p = server.params[shard]
    r = len(rows)
    if r == 0:
        return np.zeros((0, p.columnSize), np.uint64)
    pad = -r % p.chunksPerEntry
    req = np.concatenate([rows, np.zeros((pad, p.databaseColumns), server.scalar)]).reshape(-1, p.chunksPerEntry,
                                                                                          p.databaseColumns)
    single = sp.SimplePirServer(server.databases[shard], server.hints[shard], p, server.scalar)
    return single.computeResponses(req).reshape(-1, p.columnSize)[:r]


def random_rows(rng, server, shard, r, wide=False):
    p = server.params[shard]
    top = int(np.iinfo(server.scalar).max) if not wide else (1 << 64) - 1
    return rng.integers(0, top, size=(r, p.databaseColumns), dtype=np.uint64, endpoint=True).astype(server.scalar)


def check(server, messages, rows, shards):
    got = server.computeResponsesProto(messages)
    assert len(got) == len(messages)
    for j, (g, r, s) in enumerate(zip(got, rows, shards)):
        words = expected_words(server, s, r)
        want = ref.encode_response(len(r), server.params[s].columnSize, words.reshape(-1))
        assert g == want, f"message {j}"
        assert len(g) <= ref.response_capacity(len(r), server.params[s].columnSize,
                                               server.params[s].ciphertextModulusBits)
    return got


RAGGED = [(2 * 40, 1, 2, 700), (10, 3, 1, 5), (300, 1, 6, 33), (8, 1, 1, 64 * 32 * 3 + 5)]


@pytest.mark.parametrize("count", [1, 2, 16, 17])
@pytest.mark.parametrize("scalar,ct", [(np.uint32, 28), (np.uint64, 32), (np.uint64, 42), (np.uint64, 61)])
def test_byte_parity(count, scalar, ct):
    rng = np.random.default_rng(count * 100 + ct)
    server = ragged_server(rng, RAGGED, scalar, ct, 7 if ct == 28 else 14)
    shards = [int(rng.integers(0, 2)) * 2 for _ in range(count)]  # shards 1 and 3 get nothing
    rows = [random_rows(rng, server, s, int(rng.integers(0, 6))) for s in shards]
    if count > 1:
        rows[0] = rows[0][:0]  # an empty request: a 0 x M_s reply
    messages = [ref.encode_request(len(r), server.params[s].databaseColumns, r.reshape(-1), s) for r, s in zip(rows, shards)]
    got = check(server, messages, rows, shards)
    if count > 1:
        assert ref.parse_response(got[0]) == (0, server.params[shards[0]].columnSize, [])


def test_every_shard_and_ragged_traffic():
    rng = np.random.default_rng(7)
    server = ragged_server(rng, RAGGED, np.uint64, 42)
    shards = [j % 4 for j in range(40)]
    rows = [random_rows(rng, server, s, int(rng.integers(0, 9))) for s in shards]
    messages = [ref.encode_request(len(r), server.params[s].databaseColumns, r.reshape(-1), s) for r, s in zip(rows, shards)]
    check(server, messages, rows, shards)


def test_request_past_2_to_the_20_varints():
    rng = np.random.default_rng(3)
    server = ragged_server(rng, [(64, 1, 1, 4096 + 7), (10, 3, 1, 5)], np.uint64, 42)
    rows = [random_rows(rng, server, 0, 300), random_rows(rng, server, 1, 2)]
    assert rows[0].size > 1 << 20
    messages = [ref.encode_request(len(r), server.params[s].databaseColumns, r.reshape(-1), s)
                for r, s in zip(rows, [0, 1])]
    check(server, messages, rows, [0, 1])


def test_33_shards_cross_a_launch_group():
    rng = np.random.default_rng(33)
    shapes = [(10 + i, 1, 1 + i % 3, 40 + 13 * i) for i in range(33)]
    server = ragged_server(rng, shapes, np.uint64, 42)
    shards = list(range(33)) + [32, 0]
    rows = [random_rows(rng, server, s, 1 + s % 3) for s in shards]
    messages = [ref.encode_request(len(r), server.params[s].databaseColumns, r.reshape(-1), s) for r, s in zip(rows, shards)]
    check(server, messages, rows, shards)


def test_uniform_traffic_equals_the_shards_call():
    rng = np.random.default_rng(11)
    server = ragged_server(rng, RAGGED, np.uint64, 42)
    clients, per = 5, 2
    requests = [[rng.integers(0, 1 << 63, size=(per, p.chunksPerEntry, p.databaseColumns), dtype=np.uint64)
                 for p in server.params] for _ in range(clients)]
    grouped = server.computeResponses(requests)
    messages = [ref.encode_request(per * p.chunksPerEntry, p.databaseColumns, requests[c][s].reshape(-1), s)
                for c in range(clients) for s, p in enumerate(server.params)]
    got = server.computeResponsesProto(messages)
    for c in range(clients):
        for s, p in enumerate(server.params):
            rows, cols, data = ref.parse_response(got[c * len(server.params) + s])
            assert (rows, cols) == (per * p.chunksPerEntry, p.columnSize)
            assert np.array_equal(np.array(data, np.uint64), grouped[c][s].reshape(-1).astype(np.uint64)), (c, s)


@pytest.mark.parametrize("scalar", [np.uint32, np.uint64])
def test_unpacked_and_split_packed_answer_like_packed(scalar):
    rng = np.random.default_rng(5)
    ct = 28 if scalar == np.uint32 else 61
    server = ragged_server(rng, RAGGED, scalar, ct, 7 if ct == 28 else 14)
    rows = random_rows(rng, server, 0, 3)
    k = server.params[0].databaseColumns
    values = [int(v) for v in rows.reshape(-1)]
    values[:4] = [0, 127, 128, (1 << ct) - 1]
    packed = ref.encode_request(3, k, values, 0)
    forms = [ref.encode_request_with(3, k, ref.split_packed(3, values, [1, 2, 500, 1000, len(values) - 1]), 0),
             ref.encode_request_with(3, k, ref.unpacked(3, values), 0),
             ref.encode_request_with(3, k, ref.unpacked(3, values[:10]) + ref.split_packed(3, values[10:], [7]), 0)]
    got = server.computeResponsesProto([packed] + forms)
    assert all(g == got[0] for g in got[1:])
    words = np.array(values, np.uint64).astype(scalar).reshape(3, k)
    assert got[0] == ref.encode_response(3, server.params[0].columnSize, expected_words(server, 0, words).reshape(-1))


def raw_call(server, messages, fill=0xA5):
    """The C ABI call with caller-owned output, pre-filled -> (rc, error, out, lengths)."""
    lib = hecuda.load_library()
    bufs = [C.create_string_buffer(m, max(len(m), 1)) for m in messages]
    ptrs = (C.c_void_p * len(bufs))(*[C.addressof(b) for b in bufs])
    sizes = np.array([len(m) for m in messages], np.uint64)
    out = np.full(1 << 16, fill, np.uint8)
    offsets = np.arange(len(messages), dtype=np.uint64) * np.uint64(1 << 12)
    lengths = np.full(len(messages), 7, np.uint64)
    rc = lib.hecuda_simple_pir_compute_response_proto(server._h, server.shardCount, ptrs, hecuda._ptr(sizes), len(messages),
                                                      hecuda._ptr(out), hecuda._ptr(offsets), hecuda._ptr(lengths))
    return rc, (lib.hecuda_last_error() or b"").decode(), out, lengths


def test_refusals():
    rng = np.random.default_rng(9)
    server = ragged_server(rng, [(10, 3, 1, 5), (8, 1, 1, 40)], np.uint32, 28, 7)
    good = ref.encode_request(1, 5, [1, 2, 3, 4, 5], 0)
    host = [
        (b"\x0a\x05\x08", "truncated"),                                     # length past the message
        (ref.field_scalar(2, 1), "request is not set"),                    # unset request
        (ref.encode_request(1, 5, [1] * 5, 2), "shard_index 2"),            # shard_index >= shard count
        (ref.encode_request(1, 6, [1] * 6, 0), "col_count 6"),              # col_count != K_s
        (good + ref.field_bytes(1, b""), "singular message given twice"),
        (ref.field_bytes(1, ref.varint(3 << 3 | 5) + b"\0\0\0\0"), "wire type 5"),
        (ref.encode_request(1 << 31, 5, [], 0), "too large"),
    ]
    for bad, what in host:
        before = hecuda.kernel_launch_count()
        rc, err, out, lengths = raw_call(server, [good, bad])
        assert rc != 0 and err.startswith("message 1: ") and what in err, (bad, err)
        assert hecuda.kernel_launch_count() == before
        assert np.all(out == 0xA5) and np.all(lengths == 7)
    device = [
        (ref.encode_request_with(1, 5, ref.field_bytes(3, b"\x01\x02\x03\x04\x85"), 0), "runs past"),
        (ref.encode_request_with(1, 5, ref.field_bytes(3, b"\x01\x02\x03\x04" + b"\x80" * 10 + b"\x01"), 0), "longer than 10"),
        (ref.encode_request(1, 5, [1, 2, 3, 4, 1 << 32], 0), "2^32"),
        (ref.encode_request_with(1, 5, ref.packed(3, [1, 2, 3, 4]), 0), "varint count"),
        (ref.encode_request_with(1, 5, ref.packed(3, [1, 2, 3, 4, 5, 6]), 0), "varint count"),
        (ref.encode_request_with(0, 5, ref.packed(3, [1]), 0), "varint count"),
    ]
    for bad, what in device:
        rc, err, out, lengths = raw_call(server, [good, good, bad, good])
        assert rc != 0 and err.startswith("message 2: ") and what in err, (bad, err)
        assert np.all(out == 0xA5) and np.all(lengths == 7)
    # the same bytes are answered once they are whole; a 10-byte varint of 2^32 - 1 on a 32-bit shard is fine
    ten = b"\xff\xff\xff\xff\x8f\x80\x80\x80\x80\x00"
    ok = ref.encode_request_with(1, 5, ref.field_bytes(3, b"\x01\x02\x03\x04" + ten), 0)
    rc, err, out, lengths = raw_call(server, [good, ok])
    assert rc == 0, err
    words = np.array([[1, 2, 3, 4, (1 << 32) - 1]], np.uint32)
    assert bytes(out[4096:4096 + int(lengths[1])]) == ref.encode_response(1, server.params[0].columnSize,
                                                                          expected_words(server, 0, words).reshape(-1))


def test_launch_count_does_not_depend_on_the_message_count():
    rng = np.random.default_rng(13)
    server = ragged_server(rng, RAGGED, np.uint64, 42)
    counts = []
    for count in (2, 64):
        shards = [j % 4 for j in range(count)]
        messages = [ref.encode_request(2, server.params[s].databaseColumns, random_rows(rng, server, s, 2).reshape(-1), s)
                    for s in shards]
        before = hecuda.kernel_launch_count()
        server.computeResponsesProto(messages)
        counts.append(hecuda.kernel_launch_count() - before)
    assert counts[0] == counts[1] == 8, counts  # 4 decode, 1 response group, 3 encode


@pytest.mark.parametrize("scalar,pt,ct", [(np.uint32, 7, 28), (np.uint64, 14, 42)])
def test_end_to_end_from_the_tools_files(tmp_path, scalar, pt, ct):
    rng = np.random.default_rng(21)
    entries = [(i * 3 + 1, rng.integers(0, 256, size=int(rng.integers(20, 90)), dtype=np.uint8).tobytes())
               for i in range(120)]
    server = sp.SimplePirShardedServer.process(entries, enc(pt, ct, 64), 3, chunkSize=25, scalar=scalar,
                                               rng=np.random.default_rng(2))
    prefix, path = str(tmp_path / "db"), str(tmp_path / "config.binpb")
    server.save(prefix, path)
    raw = open(path, "rb").read()
    config = sp.SimplePirConfig.load(path, "unchecked")
    assert config.serialize() == raw
    assert config.databaseMap == server.databaseMap and config.params == server.params
    assert config.scalar == scalar
    import hashlib
    assert config.hintIdentifiers == [hashlib.sha256(open(f"{prefix}-{i}.hint.bin", "rb").read()).digest() for i in range(3)]
    loaded = sp.SimplePirShardedServer.fromConfig(prefix, config)
    client = sp.SimplePirClientForAllShards.fromConfig(prefix, config)
    try:
        picks = [entries[int(i)] for i in rng.choice(len(entries), 15, replace=False)] + [(2, None)]  # 2 is absent
        flows = [client.requestMessages(index) for index, _ in picks]
        flat = [m for messages, _ in flows for m in messages]
        for m in flat:
            assert sp.SimplePirRequest.fields(m)["has_request"]
        replies = loaded.computeResponsesProto(flat)
        shards = loaded.shardCount
        for c, ((index, value), (_, queries)) in enumerate(zip(picks, flows)):
            got = client.decryptResponseMessages(replies[c * shards:(c + 1) * shards], index, queries)
            assert got == value, index
    finally:
        for q in client.clients:
            q.queryGenerator.close()
        loaded.close()
        server.close()


def test_single_server_answers_shard_zero():
    rng = np.random.default_rng(17)
    prm = sp.SimplePirParameters(enc(), 80, 1, 2, 700)
    db = rng.integers(0, 1 << 14, size=(prm.columnSize, 700), dtype=np.uint64)
    server = sp.SimplePirServer(db, np.zeros((prm.columnSize, 16), np.uint64), prm)
    rows = rng.integers(0, 1 << 63, size=(4, 700), dtype=np.uint64)
    got = server.computeResponsesProto([ref.encode_request(4, 700, rows.reshape(-1), 0)])
    want = server.computeResponses(rows.reshape(2, 2, 700)).reshape(4, -1)
    assert got[0] == ref.encode_response(4, prm.columnSize, want.reshape(-1))
