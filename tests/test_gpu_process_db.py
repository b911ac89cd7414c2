"""Processing the server's own data on the GPU: MulPirServer.process (hecuda_pir_process_entries,
hecuda_pir_database_create_from_entries) and PlaintextMatrix(signedValues:) in .diagonal packing
(hecuda_pnns_diagonal_plaintexts, hecuda_pnns_matrix_create_from_values).

The host ports (plaintextRows, diagonalPlaintexts) are the reference: the device packing must equal them word for word,
the resident buffers must equal those the existing create calls build from the host packing, and the servers built
from them must answer bit-identically and decrypt to the data."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir, pnns
from oracle import oracle as orc
from oracle import pir_oracle as opir
from oracle import pnns_oracle as opn
from test_gpu_evk_wire import read_device
from test_gpu_pir_clients import CONFIGS, Setup

TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)
PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:357-367)
Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]  # C5's moduli
ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = -1, -2

# (N, moduli, t) at the three degrees the packing is checked at
CONTEXTS = {16: (16, None, 1153), 4096: (4096, PIR_MODULI, 17), 8192: (8192, Q8192, 65537)}


def context(n, scalar=np.uint64):
    n, moduli, t = CONTEXTS[n]
    moduli = moduli or orc.generate_primes(TEST_MODULI_BITS, False, n)
    return hecuda.Context(n, moduli, t, scalar=scalar)


def database(rng, entries, size, variable):
    out = []
    for i in range(entries):
        length = rng.randint(0, size) if variable else size
        out.append(bytes(length) if i % 5 == 2 else bytes(rng.randrange(256) for _ in range(length)))
    if variable and entries:
        out[-1] = bytes(rng.randrange(256) for _ in range(size))
    return out


def parameter(g, entries, size, dims, encoding, uneven=False):
    return pir.MulPir.generateParameter(pir.IndexPirConfig(entries, size, dims, 1, uneven, "noCompression", encoding), g)


# (entries, entry size, dimensions, encodingEntrySize, variable-length)
PIR_SHAPES = [(100, 1, 2, False, False), (300, 24, 1, True, True), (40, 47, 2, True, True), (500, 64, 2, False, False),
              (9, 3000, 2, True, True), (25, 9000, 1, False, False)]


@pytest.mark.parametrize("n", [16, 4096, 8192])
@pytest.mark.parametrize("shape", PIR_SHAPES)
def test_pack_entries_matches_plaintext_rows(n, shape):
    entries, size, dims, encoding, variable = shape
    g = context(n)
    param = parameter(g, entries, size, dims, encoding)
    db = database(random.Random(n + size), entries, size, variable)
    rows, present = pir.MulPirServer.plaintextRows(db, g, param)
    got_rows, got_present = pir.packEntries(db, g, param)
    assert np.array_equal(got_rows, rows)
    assert np.array_equal(got_present, present)
    g.close()


def resident_pir_words(db):
    return read_device(*db.deviceBuffer())


@pytest.mark.parametrize("n,scalar", [(16, np.uint64), (4096, np.uint64), (4096, np.uint32), (8192, np.uint64)])
@pytest.mark.parametrize("shape", PIR_SHAPES[:4])
def test_database_from_entries_is_the_host_database(n, scalar, shape):
    entries, size, dims, encoding, variable = shape
    g = context(n, scalar)
    param = parameter(g, entries, size, dims, encoding)
    db = database(random.Random(7 * n + size), entries, size, variable)
    host, device = pir.MulPirServer.process(db, g, param), pir.MulPirServer.processOnDevice(db, g, param)
    assert device.count == host.count
    host_ptr, host_bytes = host.deviceBuffer()
    dev_ptr, dev_bytes = device.deviceBuffer()
    assert dev_bytes == host_bytes
    if n == 4096:  # the 27/28-bit moduli keep uint32 rows
        assert host_bytes == host.count * g.L * n * 4
    assert np.array_equal(read_device(dev_ptr, dev_bytes), read_device(host_ptr, host_bytes))
    present = pir.MulPirServer.plaintextRows(db, g, param)[1]
    assert np.array_equal(device.presentFlags(), present) and np.array_equal(host.presentFlags(), present)
    host.close(), device.close()
    g.close()


def test_database_from_entries_spans_slabs_at_c4_parameters():
    """2^16 entries of 64 B at C4's parameters: 108 x 19 = 2052 plaintexts, more than one 64 MB slab (2048 at N = 4096)."""
    g = context(4096)
    param = parameter(g, 1 << 16, 64, 2, False, uneven=True)
    rng = np.random.default_rng(16)
    raw = rng.integers(0, 256, size=((1 << 16), 64), dtype=np.uint8)
    db = [bytes(row) for row in raw]
    host, device = pir.MulPirServer.process(db, g, param), pir.MulPirServer.processOnDevice(db, g, param)
    assert host.count > 8 * 1024 * 1024 // 4096
    assert np.array_equal(resident_pir_words(device), resident_pir_words(host))
    assert np.array_equal(device.presentFlags(), host.presentFlags())
    host.close(), device.close()
    g.close()


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("encoding", [False, True])
def test_device_processed_server_answers_like_the_host_one(cfg, encoding):
    moduli = orc.generate_primes(TEST_MODULI_BITS, False, 16)
    g, o = hecuda.Context(16, moduli, 1153), orc.Context(16, moduli, 1153)
    s = Setup(g, o, 100, cfg["entry_size"], cfg["dims"], 1, cfg["uneven"], cfg["compression"], encoding, seed=3)
    server = pir.MulPirServer(s.param, g, [pir.MulPirServer.processOnDevice(d, g, s.param) for d in s.dbs])
    for seed in (1, 2):
        c = s.client(seed)
        got = server.computeResponse(c["query"], c["key"])
        assert np.array_equal(got, s.server.computeResponse(c["query"], c["key"]))
        reply = [[got[0, chunk] for chunk in range(server.chunkCount)]]
        assert opir.decrypt_response(o, s.oparam, reply, c["indices"], c["sk"]) == [s.dbs[0][c["indices"][0]]]
        c["key"].close()
    g.close()


def _raw_pir(g, data, offsets, entry_count, entry_size, encode, dims, count=None):
    """Both PIR calls with raw arguments; returns (process rc, create rc, whether *out stayed NULL)."""
    lib = hecuda.load_library()
    dim_arr = (C.c_int32 * max(1, len(dims)))(*dims) if dims is not None else None
    d = data.ctypes.data_as(C.c_void_p) if data is not None else None
    o = offsets.ctypes.data_as(C.c_void_p) if offsets is not None else None
    h = C.c_void_p(1234)
    rc_create = lib.hecuda_pir_database_create_from_entries(g._h, d, o, entry_count, entry_size, encode, dim_arr,
                                                            len(dims or []), C.byref(h))
    stayed_null = h.value is None
    if not rc_create:
        lib.hecuda_pir_database_destroy(h)
    rows = np.zeros((max(1, count or 1), g.degree), dtype=np.uint64)
    present = np.zeros(max(1, count or 1), dtype=np.uint8)
    rc_process = lib.hecuda_pir_process_entries(g._h, d, o, entry_count, entry_size, encode, dim_arr, len(dims or []),
                                                rows.ctypes.data_as(C.c_void_p), present.ctypes.data_as(C.c_void_p),
                                                count or 1)
    return rc_process, rc_create, stayed_null


def test_pir_errors():
    import torch
    g = context(16)
    data = np.arange(40, dtype=np.uint8)
    offsets = np.array([0, 10, 20, 30, 40], dtype=np.uint64)
    # 4 entries of 10 B with t = 1153 (bytesPerPlaintext 20): 2 per plaintext, 2 plaintexts
    assert _raw_pir(g, data, offsets, 4, 10, 0, [2], 2) == (0, 0, False)
    free_before = torch.cuda.mem_get_info()[0]
    cases = {
        "null entries": (None, offsets, 4, 10, 0, [2], 2),
        "null dimensions": (data, offsets, 4, 10, 0, None, 2),
        "three dimensions": (data, offsets, 4, 10, 0, [1, 1, 2], 2),
        "no dimensions": (data, offsets, 4, 10, 0, [], 2),
        "decreasing offsets": (data, np.array([0, 10, 5, 30, 40], dtype=np.uint64), 4, 10, 0, [2], 2),
        "entry longer than entry_size": (data, np.array([0, 10, 21, 30, 40], dtype=np.uint64), 4, 10, 0, [2], 2),
        "more packed plaintexts than dimensions hold": (data, offsets, 4, 10, 0, [1], 1),
        "more split entries than dimensions hold": (data, offsets, 4, 30, 0, [1, 3], 6),
        "zero dimension": (data, offsets, 4, 10, 0, [0], 2),
    }
    for name, args in cases.items():
        rc_process, rc_create, stayed_null = _raw_pir(g, *args)
        assert rc_process == ERR_INVALID_ARGUMENT and rc_create == ERR_INVALID_ARGUMENT and stayed_null, name
    # a wrong count only concerns the process call
    assert _raw_pir(g, data, offsets, 4, 10, 0, [2], 3)[0] == ERR_INVALID_ARGUMENT
    msg = hecuda.load_library().hecuda_last_error().decode()
    assert "count" in msg
    _raw_pir(g, data, np.array([0, 10, 21, 30, 40], dtype=np.uint64), 4, 10, 0, [2], 2)
    assert "invalidDatabaseEntrySize" in hecuda.load_library().hecuda_last_error().decode()
    _raw_pir(g, data, offsets, 4, 10, 0, [1], 1)
    assert "invalidDatabaseEntryCount" in hecuda.load_library().hecuda_last_error().decode()
    with pytest.raises(pir.PirError):  # the Python layer checks entryCount as plaintextRows does
        pir.MulPirServer.processOnDevice([b"x"] * 3, g, parameter(g, 4, 1, 1, False))
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 64 << 20
    g.close()


# ---- PNNS ------------------------------------------------------------------------------------------------------------

def pnns_context(n):
    if n == 8192:
        return hecuda.Context(n, Q8192, 65537)
    bits, t = (TEST_MODULI_BITS, 97) if n == 16 else ([36, 36, 37], 65537)
    return hecuda.Context(n, orc.generate_primes(bits, False, n), t)


def signed_matrix(rng, rows, cols, t, reduce):
    if reduce:
        return rng.integers(-(1 << 50), 1 << 50, size=(rows, cols), dtype=np.int64)
    values = rng.integers(-(t // 2), (t - 1) // 2 + 1, size=(rows, cols), dtype=np.int64)
    values[0, 0] = -(t // 2)
    values[-1, -1] = (t - 1) // 2
    return values


def remainders(values, t, reduce):
    if reduce:
        return (values.reshape(-1) % t).astype(np.uint64)  # numpy's % takes the divisor's sign, as Modulus.reduce
    return pnns.centeredToRemainder(values, t).reshape(-1)


# (N, rows, cols, (babyStep, giantStep) or None)
PNNS_SHAPES = [(16, 5, 3, None), (16, 16, 5, None), (16, 37, 7, (3, 3)), (16, 40, 8, (4, 2)),
               (4096, 4095, 100, None), (4096, 4096, 64, (16, 4)), (4096, 9000, 33, (64, 1)),
               (8192, 9000, 512, None), (8192, 8192, 300, (32, 16)),
               (8192, 20000, 512, None)]  # 1536 plaintexts / 1587 resident slots: two slabs of 1024 at N = 8192


def bsgs_for(cols, steps):
    if steps is None:
        return pnns.BabyStepGiantStep.forVectorDimension(cols)
    return pnns.BabyStepGiantStep(pnns._next_power_of_two(cols), *steps)


@pytest.mark.parametrize("shape", PNNS_SHAPES)
@pytest.mark.parametrize("reduce", [False, True])
def test_diagonal_plaintexts_match_the_host_packing(shape, reduce):
    n, rows, cols, steps = shape
    g = pnns_context(n)
    t = g.plaintextModulus
    bsgs = bsgs_for(cols, steps)
    values = signed_matrix(np.random.default_rng(rows + cols), rows, cols, t, reduce)
    dims = pnns.MatrixDimensions(rows, cols)
    expected = pnns.PlaintextMatrix.diagonalPlaintexts(g, dims, bsgs, remainders(values, t, reduce))
    got = pnns.PlaintextMatrix.diagonalPlaintextsOnDevice(g, dims, bsgs, values, reduce=reduce)
    assert np.array_equal(got, expected)
    g.close()


@pytest.mark.parametrize("shape", PNNS_SHAPES)
def test_matrix_from_values_is_the_host_matrix(shape):
    n, rows, cols, steps = shape
    g = pnns_context(n)
    t = g.plaintextModulus
    bsgs = bsgs_for(cols, steps)
    values = signed_matrix(np.random.default_rng(3 * rows + cols), rows, cols, t, False)
    dims = pnns.MatrixDimensions(rows, cols)
    host = pnns.PlaintextMatrix(g, dims, remainders(values, t, False), bsgs)
    device = pnns.PlaintextMatrix.fromSignedValues(g, dims, values, bsgs)
    assert device.resultCiphertextCount == host.resultCiphertextCount
    host_ptr, host_bytes = host.deviceBuffer()
    dev_ptr, dev_bytes = device.deviceBuffer()
    assert dev_bytes == host_bytes == device.resultCiphertextCount * bsgs.giantStep * bsgs.babyStep * g.L * n * 8
    assert np.array_equal(read_device(dev_ptr, dev_bytes), read_device(host_ptr, host_bytes))
    assert np.array_equal(device.presentFlags(), host.presentFlags())
    host.close(), device.close()
    g.close()


@pytest.mark.parametrize("n,rows,cols", [(16, 10, 4), (16, 40, 5), (64, 100, 24), (4096, 5000, 128)])
def test_mul_transpose_on_a_device_processed_matrix(n, rows, cols):
    t = 1153 if n == 16 else 65537
    bits = (55, 52, 62, 58) if n == 16 else (55, 55, 55) if n == 64 else (36, 36, 37)
    moduli = orc.generate_primes(list(bits), False, n)
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    rng = np.random.default_rng(rows * 31 + cols)
    values = signed_matrix(rng, rows, cols, t, False)
    flat = remainders(values, t, False)
    dims = pnns.MatrixDimensions(rows, cols)
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(cols)
    sk, _ = o.keygen(9, relin=False)
    key, okeys = hecuda.EvaluationKey(g, None), {}
    elements = [pnns.GaloisElement.rotatingColumns(-1, n)]
    if bsgs.giantStep > 1:
        elements.append(pnns.GaloisElement.rotatingColumns(-bsgs.babyStep, n))
    for i, e in enumerate(dict.fromkeys(elements)):
        okeys[e] = o.galois_keygen(70 + i, sk, e)
        key.setGaloisKey(e, okeys[e])
    host = pnns.PlaintextMatrix(g, dims, flat, bsgs)
    device = pnns.PlaintextMatrix.fromSignedValues(g, dims, values, bsgs)
    vector = [int(v) for v in rng.integers(0, t, size=cols)]
    ct = o.encrypt(12, sk, pnns.denseRowVector(g, vector))
    got = device.mulTranspose(ct, key, modSwitchDownToSingle=True)
    assert np.array_equal(got, host.mulTranspose(ct, key, modSwitchDownToSingle=True))
    decoded = []
    for r in range(device.resultCiphertextCount):
        decoded += opn.decode_simd(o, o.decrypt(sk, got[0, r])).tolist()
    matrix = flat.reshape(rows, cols)
    assert decoded[:rows] == [sum(int(x) * y for x, y in zip(row, vector)) % t for row in matrix]
    host.close(), device.close(), key.close()
    g.close()


def _raw_pnns(g, values, reduce, rows, cols, baby, giant):
    lib = hecuda.load_library()
    v = values.ctypes.data_as(C.c_void_p) if values is not None else None
    h = C.c_void_p(1234)
    rc_create = lib.hecuda_pnns_matrix_create_from_values(g._h, v, reduce, rows, cols, baby, giant, C.byref(h))
    stayed_null = h.value is None
    if not rc_create:
        lib.hecuda_pnns_matrix_destroy(h)
    return rc_create, stayed_null


def test_pnns_errors():
    import torch
    g = pnns_context(16)  # t = 97: centered range [-48, 48]
    good = np.zeros((10, 4), dtype=np.int64)
    assert _raw_pnns(g, good, 0, 10, 4, 2, 2) == (0, False)
    bad = good.copy()
    bad[3, 2] = 49
    assert _raw_pnns(g, bad, 1, 10, 4, 2, 2) == (0, False)  # reduced: accepted
    lib = hecuda.load_library()
    free_before = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        assert _raw_pnns(g, bad, 0, 10, 4, 2, 2) == (ERR_INVALID_ARGUMENT, True)
    assert "outside" in hecuda.load_library().hecuda_last_error().decode()
    bad[3, 2] = -49
    assert _raw_pnns(g, bad, 0, 10, 4, 2, 2) == (ERR_INVALID_ARGUMENT, True)
    assert _raw_pnns(g, None, 0, 10, 4, 2, 2) == (ERR_INVALID_ARGUMENT, True)
    assert _raw_pnns(g, np.zeros((10, 9), dtype=np.int64), 0, 10, 9, 4, 4) == (ERR_INVALID_ARGUMENT, True)  # cols > N/2
    assert "invalidMatrixDimensions" in hecuda.load_library().hecuda_last_error().decode()
    assert _raw_pnns(g, good, 0, 10, 4, 1, 2) == (ERR_INVALID_ARGUMENT, True)   # babyStep < giantStep
    assert _raw_pnns(g, good, 0, 10, 4, 1, 1) == (ERR_INVALID_ARGUMENT, True)   # does not cover the dimension
    assert _raw_pnns(g, good, 0, 10, 4, 4, 2) == (ERR_INVALID_ARGUMENT, True)   # a needless giant step
    for giant in (0, -1):                                                        # no giant step at all
        assert _raw_pnns(g, good, 0, 10, 4, 4, giant) == (ERR_INVALID_ARGUMENT, True)
        coeffs = np.zeros((4, 16), dtype=np.uint64)
        h = C.c_void_p(1234)
        assert lib.hecuda_pnns_matrix_create(g._h, coeffs.ctypes.data_as(C.c_void_p), 0, 10, 4, 4, giant,
                                             C.byref(h)) == ERR_INVALID_ARGUMENT and h.value is None
    out = np.zeros((4, 16), dtype=np.uint64)
    assert lib.hecuda_pnns_diagonal_plaintexts(g._h, bad.ctypes.data_as(C.c_void_p), 0, 10, 4, 2,
                                               out.ctypes.data_as(C.c_void_p)) == ERR_INVALID_ARGUMENT
    assert lib.hecuda_pnns_diagonal_plaintexts(g._h, good.ctypes.data_as(C.c_void_p), 0, 10, 4, 0,
                                               out.ctypes.data_as(C.c_void_p)) == ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 64 << 20
    g.close()
    # t = 17 is not 1 mod 2N: no SIMD encoding
    plain = hecuda.Context(16, orc.generate_primes(TEST_MODULI_BITS, False, 16), 17)
    assert _raw_pnns(plain, good, 0, 10, 4, 2, 2) == (ERR_UNSUPPORTED, True)
    with pytest.raises(hecuda.HeError):
        pnns.PlaintextMatrix.fromSignedValues(plain, pnns.MatrixDimensions(10, 4), good)
    plain.close()


def test_large_matrix_leaks_nothing_on_a_bad_value():
    """A C5-sized matrix that fails its range check frees everything it allocated (about 0.4 GB each)."""
    import torch
    g = pnns_context(8192)
    rows, cols = 20000, 512
    values = np.zeros((rows, cols), dtype=np.int64)
    values[-1, -1] = 1 << 40
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(cols)
    free_before = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        assert _raw_pnns(g, values, 0, rows, cols, bsgs.babyStep, bsgs.giantStep) == (ERR_INVALID_ARGUMENT, True)
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 256 << 20
    g.close()
