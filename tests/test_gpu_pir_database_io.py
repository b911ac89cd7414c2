"""Saving and loading processed PIR databases on the GPU (hecuda_pir_databases_serialize,
hecuda_pir_databases_create_serialized): the reference's ProcessedDatabase file format, packed and unpacked on the
device.

The restatement in tests/pir_database_io_ref.py (pinned on a known-answer test) is the reference for every byte; a
loaded database must be word for word the one hecuda_pir_database_create_from_entries builds, and a server over it must
answer exactly as the original."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import keyword_pir as kw
from hecuda import pir
from hecuda import symmetric_pir as sp
import pir_database_io_ref as ref
from oracle import pir_oracle as opir
from test_gpu_evk_wire import read_device
from test_gpu_process_db import PIR_MODULI, context, database, parameter

ERR_INVALID_ARGUMENT = -1


def lib():
    return hecuda.load_library()


def last_error():
    return lib().hecuda_last_error().decode()


def oracle_bytes(g, db, param):
    """The reference serialization of the host path's Eval plaintexts: plaintextRows, then plaintextToEval."""
    rows, present = pir.MulPirServer.plaintextRows(db, g, param)
    evals = hecuda.Bfv.plaintextToEval(g, rows)
    return ref.serialize_processed_database(g.degree, g.ciphertextModuli,
                                            [evals[i] if present[i] else None for i in range(len(present))])


def resident(db):
    return read_device(*db.deviceBuffer()), db.presentFlags()


def same_database(a, b):
    wa, pa = resident(a)
    wb, pb = resident(b)
    return a.count == b.count and np.array_equal(wa, wb) and np.array_equal(pa, pb)


def first_difference(a, b):
    a, b = np.frombuffer(bytes(a), dtype=np.uint8), np.frombuffer(bytes(b), dtype=np.uint8)
    n = min(a.size, b.size)
    diff = np.flatnonzero(a[:n] != b[:n])
    return (int(diff[0]) if diff.size else n, a.size, b.size)


# (N, entries, entry size, dimensions): the 4096 shapes keep uint32 rows, the 8192 one uint64.  The all-zero entries
# (every fifth) and the padding to prod(dimensions) give nil plaintexts.
SHAPES = [(16, 100, 24, 2), (4096, 300, 64, 2), (4096, 200, 1000, 1), (8192, 150, 3000, 2)]


@pytest.mark.parametrize("n,entries,size,dims", SHAPES)
def test_save_is_the_reference_serialization(n, entries, size, dims):
    g = context(n)
    param = parameter(g, entries, size, dims, False)
    db = database(random.Random(n + size), entries, size, False)
    processed = pir.MulPirServer.processOnDevice(db, g, param)
    expected = oracle_bytes(g, db, param)
    assert processed.serializationByteCount() == len(expected)
    got = processed.serialize()
    assert got == expected, first_difference(got, expected)
    # load: word for word the database processed from the entries
    loaded, = pir.ProcessedDatabase.load(g, expected)
    assert same_database(loaded, processed)
    loaded.close(), processed.close()
    g.close()


def test_uint32_context_reads_and_writes_the_same_bytes():
    g64, g32 = context(4096), context(4096, np.uint32)
    param = parameter(g64, 300, 64, 2, False)
    db = database(random.Random(5), 300, 64, False)
    a, b = pir.MulPirServer.processOnDevice(db, g64, param), pir.MulPirServer.processOnDevice(db, g32, param)
    data = a.serialize()
    assert b.serialize() == data
    loaded, = pir.ProcessedDatabase.load(g32, data)
    assert same_database(loaded, b)
    for x in (a, b, loaded):
        x.close()
    g64.close(), g32.close()


def test_round_trip_serves_the_same_responses(tmp_path):
    g = context(4096)
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(500, 40, 2, 1, False, "hybridCompression", True), g)
    db = database(random.Random(9), 500, 40, True)
    original = pir.MulPirServer(param, g, [pir.MulPirServer.processOnDevice(db, g, param)])
    path = str(tmp_path / "shard.bin")
    original.databases[0].save(path)
    with open(path, "rb") as f:
        assert f.read() == original.databases[0].serialize()
    server = pir.MulPirServer.load(path, param, g)
    assert same_database(server.databases[0], original.databases[0])
    client = pir.MulPirClient(param, g)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    for index in (0, 123, 499):
        query = client.generateQuery([index], sk)
        response = server.computeResponse(query, key)
        assert np.array_equal(response, original.computeResponse(query, key))
        assert client.decrypt(response, [index], sk) == [db[index]]
    assert server.validate((77, db[77])).decryptedRow == db[77]
    wrong = pir.MulPir.generateParameter(pir.IndexPirConfig(5000, 40, 2, 1, False, "hybridCompression", True), g)
    with pytest.raises(pir.PirError, match="invalidDatabasePlaintextCount"):
        pir.MulPirServer.load(path, wrong, g)
    key.close()
    for d in server.databases + original.databases:
        d.close()
    g.close()


@pytest.mark.parametrize("symmetric", [False, True])
def test_keyword_shard_round_trip(tmp_path, symmetric):
    g = hecuda.Context(4096, PIR_MODULI, 17)
    r = random.Random(12)
    rows = [(bytes(r.randrange(256) for _ in range(12)), bytes(r.randrange(256) for _ in range(r.choice((1, 20, 60)))))
            for _ in range(300)]
    config = sp.SymmetricPirConfig(random.Random(20).randrange(1, 1 << 300).to_bytes(48, "big")) if symmetric else None
    served = kw.KeywordDatabase.symmetricPIRProcess(rows, config) if symmetric else rows
    kconfig = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(150), False, "noCompression")
    processed = kw.KeywordPirServer.processOnDevice(served, kconfig, g, kw.Rng.counter(4), symmetricPirConfig=config)
    path = str(tmp_path / "keyword.bin")
    processed.save(path)
    with open(path, "rb") as f:
        data = f.read()
    plaintexts = []
    for d in processed.databases:
        words, flags = resident(d)
        rows32 = words.view(np.uint32).reshape(d.count, g.L, g.degree).astype(np.uint64)
        plaintexts += [rows32[i] if flags[i] else None for i in range(d.count)]
    assert data == ref.serialize_processed_database(g.degree, g.ciphertextModuli, plaintexts)
    loaded = kw.ProcessedKeywordDatabase.load(path, g, processed.pirParameter, kconfig.parameter, config)
    assert loaded.table is None and loaded.symmetricPirConfig is config
    assert len(loaded.databases) == kconfig.parameter.hashFunctionCount
    for a, b in zip(loaded.databases, processed.databases):
        assert same_database(a, b)
    server = kw.KeywordPirServer(g, loaded)
    client = kw.KeywordPirClient(kconfig.parameter, processed.pirParameter, g)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    for keyword, value in served[:3] + [(b"absent keyword", None)]:
        assert client.decrypt(server.computeResponse(client.generateQuery(keyword, sk), key), keyword, sk) == value
    key.close()
    loaded.close(), processed.close()
    g.close()


@pytest.mark.parametrize("pinned", [False, True])
def test_streams_a_database_larger_than_two_chunks(tmp_path, pinned):
    """6 000 plaintexts at N = 4096 over the two 27/28-bit ciphertext moduli (about 170 MB): more than two 64 MB
    staging chunks each way."""
    g = context(4096)
    count = 6000
    rng = np.random.default_rng(4)
    rows = np.zeros((count, g.L, g.degree), dtype=np.uint64)
    for i, q in enumerate(g.ciphertextModuli):
        rows[:, i, :] = rng.integers(0, q, size=(count, g.degree), dtype=np.uint64)
    rows[:, :, 0] = np.array(g.ciphertextModuli, dtype=np.uint64) - 1
    present = (np.arange(count) % 97 != 5).astype(np.uint8)
    rows[present == 0] = 0
    original = pir.ProcessedDatabase(g, rows, present, evalFormat=True)
    expected = ref.serialize_processed_database(g.degree, g.ciphertextModuli,
                                                [rows[i] if present[i] else None for i in range(count)])
    assert len(expected) > 2 * (64 << 20)
    if pinned:
        buf = hecuda.PinnedBuffer((len(expected),), np.uint8)
        out = buf.array
    else:
        out = np.empty(len(expected), dtype=np.uint8)
    written = C.c_uint64(0)
    handles = (C.c_void_p * 1)(original._h)
    assert lib().hecuda_pir_databases_serialize(handles, 1, out.ctypes.data_as(C.c_void_p), out.size, C.byref(written)) == 0
    assert written.value == len(expected) and out.tobytes() == expected, first_difference(out, expected)
    source = out if pinned else str(tmp_path / "big.bin")
    if not pinned:
        original.save(source)
    loaded, = pir.ProcessedDatabase.load(g, source)
    assert same_database(loaded, original)
    loaded.close(), original.close()
    if pinned:
        buf.free()
    g.close()


# ---- refusals ------------------------------------------------------------------------------------------------------

def raw_load(g, data, tables=1):
    buf = np.frombuffer(bytes(data) or b"\0", dtype=np.uint8)
    handles = (C.c_void_p * tables)(*([1234] * tables))
    rc = lib().hecuda_pir_databases_create_serialized(g._h, buf.ctypes.data_as(C.c_void_p), len(data), tables, handles)
    stayed_null = all(h is None for h in handles)
    if rc == 0:
        for h in handles:
            lib().hecuda_pir_database_destroy(h)
    return rc, stayed_null


def test_refusals():
    import torch
    g = context(16)
    param = parameter(g, 100, 24, 2, False)
    db = pir.MulPirServer.processOnDevice(database(random.Random(1), 100, 24, False), g, param)
    data = db.serialize()
    size = opir.serialization_byte_count(16, g.ciphertextModuli)
    flags = db.presentFlags()
    tags = np.cumsum([5] + [1 + (size if f else 0) for f in flags])
    first_present = int(np.argmax(flags))
    last_present = int(len(flags) - 1 - np.argmax(flags[::-1]))
    count = db.count
    assert raw_load(g, data) == (0, False)
    assert raw_load(g, data + b"\x09" * 100) == (0, False)  # trailing bytes are accepted
    assert raw_load(g, data, 2)[0] == (0 if count % 2 == 0 else ERR_INVALID_ARGUMENT)
    free_before = torch.cuda.mem_get_info()[0]
    tag1 = int(tags[1])
    cases = {
        "invalidDatabaseSerializationVersion(serializationVersion: 2, expected: 1)": b"\x02" + data[1:],
        "invalidDatabaseSerializationPlaintextTag(tag: 7)": data[:tag1] + b"\x07" + data[tag1 + 1:],
        "corruptedData(the header": data[:3],
        "corruptedData(plaintextCount": data[:1] + (10 ** 6).to_bytes(4, "little") + data[5:],
        f"corruptedData(plaintext {last_present} ": data[:int(tags[last_present]) + 1 + size // 2],
        f"corruptedData(plaintext {count - 1} ": data[:-1],
        "invalidDatabasePlaintextCount": None,
        "emptyDatabase": b"\x01\x00\x00\x00\x00",
    }
    for message, raw in cases.items():
        before = hecuda.kernel_launch_count()
        rc, stayed_null = raw_load(g, raw) if raw is not None else raw_load(g, data, count + 1)
        assert rc == ERR_INVALID_ARGUMENT and stayed_null, message
        assert message in last_error(), (message, last_error())
        assert hecuda.kernel_launch_count() == before, message
    # a residue >= its modulus: found on the device, named by plaintext and row
    start = int(tags[first_present]) + 1
    bad = bytearray(data)
    bad[start:start + 7] = b"\xff" * 7  # coefficient 0 of row 0 becomes 2^ceil(log2 q_0) - 1 >= q_0
    assert raw_load(g, bytes(bad)) == (ERR_INVALID_ARGUMENT, True)
    assert f"corruptedData(plaintext {first_present}, row 0" in last_error()
    # saving
    handles = (C.c_void_p * 2)(db._h, None)
    out = np.zeros(len(data), dtype=np.uint8)
    written = C.c_uint64(99)
    before = hecuda.kernel_launch_count()
    assert lib().hecuda_pir_databases_serialize(handles, 1, out.ctypes.data_as(C.c_void_p), len(data) - 1,
                                                C.byref(written)) == ERR_INVALID_ARGUMENT
    assert "capacity" in last_error() and written.value == 0
    assert lib().hecuda_pir_databases_serialize(handles, 2, out.ctypes.data_as(C.c_void_p), len(data),
                                                C.byref(written)) == ERR_INVALID_ARGUMENT
    other = context(16)
    foreign = pir.ProcessedDatabase(other, np.zeros((2, other.L, 16), dtype=np.uint64), evalFormat=True)
    handles[1] = foreign._h
    assert lib().hecuda_pir_databases_serialize(handles, 2, out.ctypes.data_as(C.c_void_p), len(data),
                                                C.byref(written)) == ERR_INVALID_ARGUMENT
    assert "different contexts" in last_error()
    empty = pir.ProcessedDatabase(g, np.zeros((3, g.L, 16), dtype=np.uint64), np.zeros(3, dtype=np.uint8), evalFormat=True)
    with pytest.raises(hecuda.HeError, match="emptyDatabase"):
        empty.serialize()
    assert hecuda.kernel_launch_count() == before
    for x in (foreign, empty, db):
        x.close()
    other.close()
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 64 << 20
    g.close()


def test_large_load_leaks_nothing_on_a_bad_residue():
    """A C4-sized file (32 775 plaintexts at N = 4096, about 0.92 GB) whose last residue is out of range frees
    everything the load allocated: 1.07 GB of rows and the staging buffers."""
    import torch
    g = context(4096)
    size = opir.serialization_byte_count(4096, g.ciphertextModuli)  # rows of 27 and 28 bits
    count = 32775
    data = np.zeros(5 + count * (1 + size), dtype=np.uint8)
    data[0] = 1
    data[1:5] = np.frombuffer(count.to_bytes(4, "little"), dtype=np.uint8)
    data[5::1 + size] = 1
    data[-4:] = 0xff  # the last coefficient of the last row: 2^28 - 1 >= q_1
    free_before = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        with pytest.raises(hecuda.HeError, match=f"corruptedData\\(plaintext {count - 1}, row 1"):
            pir.ProcessedDatabase.load(g, data)
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 256 << 20
    g.close()
