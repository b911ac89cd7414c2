"""Saving and loading processed PNNS databases on the GPU (hecuda_pnns_database_serialize,
hecuda_pnns_matrices_create_serialized): the reference's SerializedProcessedDatabase protobuf file, packed and unpacked
on the device.

The restatement in tests/pnns_database_io_ref.py (pinned by a known-answer test and google.protobuf) is the reference
for every byte; a loaded matrix must be word for word and flag for flag the one it was saved from, and a server over it
must answer exactly as the original."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pnns
from oracle import oracle as orc
from oracle import pir_oracle as opir

import pnns_database_io_ref as ref
from test_gpu_pnns_client import Q8192, config_for, contexts, database, read_device, seeds

OK, INVALID, UNSUPPORTED = 0, -1, -2


def lib():
    return hecuda.load_library()


def config_dict(sc: pnns.ServerConfig) -> dict:
    cc = sc.clientConfig
    p = cc.encryptionParameters[0]
    b = sc.babyStepGiantStep
    return {"client_config": {
        "encryption_parameters": {"polynomial_degree": p.polyDegree, "plaintext_modulus": p.plaintextModulus,
                                  "coefficient_moduli": list(p.coefficientModuli), "he_scheme": 1,
                                  "error_std_dev": 1 if cc.errorStdDev == 6.4 else 0,
                                  "security_level": 1 if cc.securityLevel == "quantum128" else 0},
        "scaling_factor": cc.scalingFactor, "query_packing": ("denseRow",), "vector_dimension": cc.vectorDimension,
        "galois_elements": list(cc.evaluationKeyConfig.galoisElements), "extra_plaintext_moduli": cc.extraPlaintextModuli},
        "database_packing": ("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))}


def resident(m):
    return read_device(*m.deviceBuffer()), m.presentFlags()


def same_matrices(a, b):
    for x, y in zip(a.plaintextMatrices, b.plaintextMatrices):
        wx, px = resident(x)
        wy, py = resident(y)
        if not (np.array_equal(wx, wy) and np.array_equal(px, py) and x.resultCiphertextCount == y.resultCiphertextCount
                and x.babyStepGiantStep == y.babyStepGiantStep and x.dimensions == y.dimensions):
            return False
    return len(a.plaintextMatrices) == len(b.plaintextMatrices)


def restatement(processed: pnns.ProcessedDatabase, polys) -> bytes:
    d = processed.plaintextMatrices[0].dimensions
    b = processed.serverConfig.babyStepGiantStep
    matrices = [{"num_rows": d.rowCount, "num_columns": d.columnCount, "plaintexts": p,
                 "packing": ("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))} for p in polys]
    return ref.encode_processed_database(matrices, processed.entryIds, processed.entryMetadatas,
                                         config_dict(processed.serverConfig))


def first_difference(a, b):
    a, b = np.frombuffer(bytes(a), dtype=np.uint8), np.frombuffer(bytes(b), dtype=np.uint8)
    n = min(a.size, b.size)
    diff = np.flatnonzero(a[:n] != b[:n])
    return (int(diff[0]) if diff.size else n, a.size, b.size)


def signed_database(n, moduli, ts, rows, cols, metadata, seed):
    """fromSignedValues matrices and the restatement's polys from the oracle's diagonal packing and NTT."""
    gs, os_ = contexts(n, moduli, ts)
    cc, sc = config_for(n, moduli, ts, rows, cols, 1, s=100)
    rng = np.random.default_rng(seed)
    values = rng.integers(-30000, 30000, size=(rows, cols), dtype=np.int64)
    dims = pnns.MatrixDimensions(rows, cols)
    reduce = len(ts) > 1
    matrices = [pnns.PlaintextMatrix.fromSignedValues(g, dims, values, sc.babyStepGiantStep, reduce=reduce) for g in gs]
    polys = [ref.diagonal_polys(o, rows, cols, [int(v) % t for v in values.ravel()],
                                (sc.babyStepGiantStep.vectorDimension, sc.babyStepGiantStep.babyStep,
                                 sc.babyStepGiantStep.giantStep)) for o, t in zip(os_, ts)]
    meta = [bytes([i % 251]) * (i % 3) for i in range(rows)] if metadata else []
    ids = [int(v) for v in rng.integers(0, 1 << 63, rows, dtype=np.uint64)]
    return pnns.ProcessedDatabase(gs, matrices, ids, meta, sc), polys


# (N, coefficient moduli, plaintext moduli count, rows, cols, metadata)
SIGNED = [(4096, "36x3", 1, 300, 64, True), (4096, "36x3", 3, 300, 100, False), (8192, "c5", 1, 100, 64, False),
          (8192, "c5", 3, 9000, 20, True)]


def moduli_for(n, kind):
    return Q8192 if kind == "c5" else orc.generate_primes([36, 36, 37], False, n)


def plaintext_moduli(n, count):
    return [65537] + orc.generate_primes([20, 20], True, n)[:count - 1]


@pytest.mark.parametrize("n,kind,tcount,rows,cols,metadata", SIGNED)
def test_save_of_signed_values_is_the_restatement(n, kind, tcount, rows, cols, metadata):
    processed, polys = signed_database(n, moduli_for(n, kind), plaintext_moduli(n, tcount), rows, cols, metadata, n + rows)
    expected = restatement(processed, polys)
    assert processed.serializationByteCount() == len(expected)
    got = processed.serialize()
    assert got == expected, first_difference(got, expected)
    loaded = pnns.ProcessedDatabase.load(expected, processed.contexts)
    assert same_matrices(loaded, processed)
    assert loaded.entryIds == processed.entryIds and loaded.entryMetadatas == processed.entryMetadatas
    loaded.close(), processed.close()


@pytest.mark.parametrize("tcount,metadata", [(1, True), (3, False)])
def test_save_of_processed_vectors_is_the_restatement(tcount, metadata):
    n, rows, cols = 8192, 300, 128
    ts = plaintext_moduli(n, tcount)
    gs, _ = contexts(n, Q8192, ts)
    cc, sc = config_for(n, Q8192, ts, rows, cols, 4)
    vectors = np.random.default_rng(3).standard_normal((rows, cols)).astype(np.float32)
    db = database(vectors)
    if not metadata:
        db = pnns.Database([pnns.DatabaseRow(r.entryId, b"", r.vector) for r in db.rows])
    processed = pnns.ProcessedDatabase.processOnDevice(db, sc, gs)
    b = sc.babyStepGiantStep
    polys = [ref.polys_from_resident(n, Q8192[:3], resident(m)[0], rows, cols, (b.vectorDimension, b.babyStep, b.giantStep))
             for m in processed.plaintextMatrices]
    expected = restatement(processed, polys)
    assert processed.serialize() == expected
    loaded = pnns.ProcessedDatabase.load(expected)  # contexts made from the config
    assert same_matrices(loaded, processed)
    assert [g.plaintextModulus for g in loaded.contexts] == ts
    loaded.close(), processed.close()


def test_round_trip_serves_the_same_replies(tmp_path):
    n, rows, cols, q = 8192, 2000, 512, 4
    ts = plaintext_moduli(n, 2)
    gs, _ = contexts(n, Q8192, ts)
    cc, sc = config_for(n, Q8192, ts, rows, cols, q)
    vectors = np.random.default_rng(8).standard_normal((rows, cols)).astype(np.float32)
    original = pnns.ProcessedDatabase.processOnDevice(database(vectors), sc, gs)
    path = str(tmp_path / "processed.binpb")
    original.save(path)
    with open(path, "rb") as f:
        assert f.read() == original.serialize()
    loaded = pnns.ProcessedDatabase.load(path)
    assert same_matrices(loaded, original)
    assert loaded.entryIds == original.entryIds and loaded.entryMetadatas == original.entryMetadatas
    client = pnns.Client(cc, gs)
    servers = [pnns.Server(original), pnns.Server(loaded)]
    sk = client.generateSecretKey(seed=bytes(32))
    key = client.generateEvaluationKey(sk)
    count = pnns.CiphertextMatrix.ciphertextCount(n, pnns.MatrixDimensions(q, cols))
    a = [seeds(("a", k), count) for k in range(len(ts))]
    e = [seeds(("e", k), count) for k in range(len(ts))]
    query = client.generateQuery(vectors[:q], sk, aSeeds=a, errorSeeds=e)
    wire = client.generateQuery(vectors[:q], sk, wire=True, aSeeds=a, errorSeeds=e)
    r0, r1 = (s.computeResponse(query, key) for s in servers)
    for x, y in zip(r0.ciphertextMatrices, r1.ciphertextMatrices):
        assert np.array_equal(x, y)
    d0, d1 = client.decrypt(r0, sk), client.decrypt(r1, sk)
    assert np.array_equal(d0.distances, d1.distances) and d1.entryIds == d0.entryIds
    many = [s.computeResponses([query, query], [key, key]) for s in servers]
    for x, y in zip(many[0][1].ciphertextMatrices, many[1][1].ciphertextMatrices):
        assert np.array_equal(x, y)
    w0, w1 = (s.computeResponse(wire, key) for s in servers)
    for x, y in zip(w0.ciphertextMatrices, w1.ciphertextMatrices):
        assert np.array_equal(x[0], y[0])
    assert np.array_equal(client.decrypt(w1, sk).distances, client.decrypt(w0, sk).distances)
    assert loaded.validate(vectors[:2]).noiseBudget > 0
    key.close(), loaded.close(), original.close()


def big_database():
    """N = 8192, 16 384 rows of 512 columns: 1 024 plaintexts of 165 KB (173 MB), three 64 MB chunks."""
    n, rows, cols = 8192, 16384, 512
    gs, _ = contexts(n, Q8192, [65537])
    cc, sc = config_for(n, Q8192, [65537], rows, cols, 1, s=100)
    values = np.random.default_rng(12).integers(-32768, 32768, size=(rows, cols), dtype=np.int64)
    m = pnns.PlaintextMatrix.fromSignedValues(gs[0], pnns.MatrixDimensions(rows, cols), values, sc.babyStepGiantStep)
    return pnns.ProcessedDatabase(gs, [m], list(range(rows)), [], sc)


def test_loads_from_every_source(tmp_path):
    original = big_database()
    data = original.serialize()
    assert len(data) > 2 * (64 << 20)
    pinned = hecuda.PinnedBuffer((len(data),), np.uint8)
    pinned.array[:] = np.frombuffer(data, dtype=np.uint8)
    path = str(tmp_path / "big.binpb")
    original.save(path)
    for source in (data, pinned.array, np.frombuffer(data, dtype=np.uint8).copy(), path):
        loaded = pnns.ProcessedDatabase.load(source, original.contexts)
        assert same_matrices(loaded, original)
        loaded.close()
    # a save into a pinned buffer equals the pageable one
    out = hecuda.PinnedBuffer((len(data),), np.uint8)
    original._serialize_into(out.array)
    assert out.array.tobytes() == data
    pinned.free(), out.free()
    original.close()


def test_configs_round_trip():
    n = 8192
    ts = plaintext_moduli(n, 3)
    cc, sc = config_for(n, Q8192, ts, 1000, 512, 16)
    data = sc.serialize()
    assert data == ref.encode_server_config(config_dict(sc))
    back = pnns.ServerConfig.deserialize(data)
    assert back.serialize() == data and back.babyStepGiantStep == sc.babyStepGiantStep
    assert back.plaintextModuli == ts and back.evaluationKeyConfig.galoisElements == cc.evaluationKeyConfig.galoisElements
    client = cc.serialize()
    assert client == ref.encode_client_config(config_dict(sc)["client_config"])
    assert pnns.ClientConfig.deserialize(client).serialize() == client
    # stdDev64 and quantum128 survive the round trip; C5's 220 bits at N = 8192 cannot claim quantum128
    p = pnns.EncryptionParameters(4096, 65537, tuple(orc.generate_primes([27, 27, 28], False, 4096)))
    secure = pnns.ClientConfig(p, 10, 64, cc.evaluationKeyConfig, securityLevel="quantum128")
    assert pnns.ClientConfig.deserialize(secure.serialize()).securityLevel == "quantum128"
    wide = pnns.ClientConfig(p, 10, 64, cc.evaluationKeyConfig, errorStdDev=6.4)
    assert pnns.ClientConfig.deserialize(wide.serialize()).errorStdDev == 6.4
    with pytest.raises(pnns.PnnsError, match="insecureEncryptionParameters"):
        pnns.ClientConfig(cc.encryptionParameters[0], 10, 64, cc.evaluationKeyConfig, securityLevel="quantum128")
    claim = config_dict(sc)
    claim["client_config"]["encryption_parameters"]["security_level"] = 1
    with pytest.raises(pnns.PnnsError, match="insecureEncryptionParameters"):
        pnns.ServerConfig.deserialize(ref.encode_server_config(claim))
    # a server needs no sampler: a stdDev64 database serves, but the device client cannot encrypt for it
    gs, _ = contexts(4096, list(p.coefficientModuli), [65537])
    with pytest.raises(hecuda.HeError, match="errorStdDev"):
        pnns.Client(wide, gs)


def raw_load(gs, data):
    buf = np.frombuffer(bytes(data) or b"\0", dtype=np.uint8)
    handles = (C.c_void_p * len(gs))(*([1234] * len(gs)))
    ctxs = (C.c_void_p * len(gs))(*[g._h.value for g in gs])
    rc = lib().hecuda_pnns_matrices_create_serialized(ctxs, len(gs), buf.ctypes.data_as(C.c_void_p), len(bytes(data)), handles)
    stayed_null = all(h is None for h in handles)
    if rc == OK:
        for h in handles:
            lib().hecuda_pnns_matrix_destroy(h)
    return rc, stayed_null


def test_refusals_launch_nothing():
    import torch
    n, rows, cols = 4096, 300, 64
    ts = plaintext_moduli(n, 2)
    processed, polys = signed_database(n, moduli_for(n, "36x3"), ts, rows, cols, True, 5)
    gs = processed.contexts
    data = processed.serialize()
    assert raw_load(gs, data) == (OK, False)
    cfg = config_dict(processed.serverConfig)
    d = processed.plaintextMatrices[0].dimensions
    b = processed.serverConfig.babyStepGiantStep

    def rebuild(polys=polys, cfg=cfg, packing=("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))):
        ms = [{"num_rows": d.rowCount, "num_columns": d.columnCount, "plaintexts": p, "packing": packing} for p in polys]
        return ref.encode_processed_database(ms, processed.entryIds, processed.entryMetadatas, cfg)

    assert rebuild() == data
    bgv = config_dict(processed.serverConfig)
    bgv["client_config"]["encryption_parameters"]["he_scheme"] = 2
    dense = config_dict(processed.serverConfig)
    dense["database_packing"] = ("denseRow",)
    one_extra_more = config_dict(processed.serverConfig)
    one_extra_more["client_config"]["extra_plaintext_moduli"] = ts[1:] + [ts[1]]
    cases = [
        ("truncated(", data[:-3], gs, INVALID),
        ("unsetField(SerializedProcessedDatabase.serverConfig)",
         b"".join(ref.message(f, v) for f, _, v in ref.fields(data) if f != 4), gs, INVALID),
        ("invalidScheme", rebuild(cfg=bgv), gs, INVALID),
        ("only .diagonal", rebuild(packing=("denseRow",)), gs, UNSUPPORTED),
        ("only .diagonal", rebuild(cfg=dense), gs, UNSUPPORTED),
        ("wrongPlaintextCount(got: 63, expected: 64)", rebuild(polys=[p[:-1] for p in polys]), gs, INVALID),
        ("bytes of poly", rebuild(polys=[p[:-1] + [p[-1][:-1]] for p in polys]), gs, INVALID),
        ("wrongContextsCount(got: 2, expected: 3)", rebuild(cfg=one_extra_more), gs, INVALID),
        ("wrongEncryptionParameters", data, gs[::-1], INVALID),
        ("malformedProtobuf", ref.key(1, 0) + ref.varint(1) + data, gs, INVALID),
    ]
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    for message, raw, ctxs, code in cases:
        before = hecuda.kernel_launch_count()
        rc, stayed_null = raw_load(ctxs, raw)
        assert rc == code and stayed_null, (message, rc, lib().hecuda_last_error().decode())
        assert message in lib().hecuda_last_error().decode(), (message, lib().hecuda_last_error().decode())
        assert hecuda.kernel_launch_count() == before, message
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 16 << 20
    # saving with a config that does not match the matrices
    before = hecuda.kernel_launch_count()
    wrong = pnns.ProcessedDatabase(gs, processed.plaintextMatrices, processed.entryIds, processed.entryMetadatas,
                                   config_for(n, moduli_for(n, "36x3"), ts[:1], rows, cols, 1, s=100)[1])
    with pytest.raises(hecuda.HeError, match="wrongContextsCount"):
        wrong.serialize()
    assert hecuda.kernel_launch_count() == before
    processed.close()


def test_failed_residue_check_frees_everything():
    """A three-chunk file whose last plaintext has a residue >= q_2 is refused by the device-side check, naming the
    matrix, plaintext and row, and device memory returns to its level before the call."""
    import torch
    original = big_database()
    data = bytearray(original.serialize())
    gs = original.contexts
    walk = ref.parse_processed_database(bytes(data))
    count = len(walk["matrices"][0]["plaintexts"])
    poly_bytes = opir.serialization_byte_count(8192, Q8192[:3])
    end = len(data) - len(ref.message(4, ref.encode_server_config(config_dict(original.serverConfig)))) \
        - len(ref.packed(2, original.entryIds))
    b = original.serverConfig.babyStepGiantStep
    packing = ref.message(4, ref.encode_packing(("diagonal", (b.vectorDimension, b.babyStep, b.giantStep))))
    last_poly_end = end - len(packing)  # the matrix ends with its packing
    data[last_poly_end - 7:last_poly_end] = b"\xff" * 7  # the last coefficient of row 2: 2^55 - 1 >= q_2
    original.close()
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    with pytest.raises(hecuda.HeError, match=f"corruptedData\\(matrix 0, plaintext {count - 1}, row 2"):
        pnns.ProcessedDatabase.load(bytes(data), gs)
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 64 << 20
    assert poly_bytes * count < len(data)
