"""SimplePIR on the GPU (hecuda.simple_pir over csrc/simple_pir.cu) against oracle/simple_pir_oracle.py: the processed
database and hint bit-exact, responses bit-exact at random full-width words and at the accumulator bounds, batched and
device-pointer calls, noiseless end-to-end retrieval, save/load, and the refusals."""
import random

import numpy as np
import pytest

import hecuda
from hecuda import simple_pir as sp
from hecuda.pir import PirError
from oracle import simple_pir_oracle as osp

pytestmark = pytest.mark.gpu


def enc(pt, ct, n, std=3.2):
    return sp.SimplePirEncryptionParams(pt, ct, n, std, "unchecked")


def raw(rng, count, size):
    return np.array([[rng.randrange(256) for _ in range(size)] for _ in range(count)], dtype=np.uint8)


def processed(entries, prm):
    return osp.process_database(entries, prm.plaintextModulusBits, prm.entriesPerColumn, prm.chunksPerEntry,
                                prm.databaseColumns)


SHAPES = [  # pt, ct, N, entries, size, scalar
    (7, 28, 8, 600, 20, np.uint32), (14, 42, 16, 600, 20, np.uint64), (7, 28, 8, 20, 600, np.uint32),
    (14, 42, 16, 20, 600, np.uint64), (14, 42, 1024, 3000, 40, np.uint64), (14, 42, 2048, 5000, 24, np.uint64),
    (14, 42, 16, 40, 600, np.uint64),  # aPolyCount > 1 and chunksPerEntry > 1
    # the reference's noiselessSample shapes: 10- and 9-bit moduli p through the small-degree NTT
    (8, 9, 16, 1, 1, np.uint32), (8, 9, 8, 10, 1, np.uint32), (4, 8, 8, 1, 1, np.uint32), (4, 8, 8, 10, 62, np.uint64),
]


@pytest.mark.parametrize("pt,ct,n,count,size,scalar", SHAPES)
def test_process_is_bit_exact(pt, ct, n, count, size, scalar):
    rng = random.Random(count * size + n)
    entries = raw(rng, count, size)
    res = sp.SimplePirServer.process(entries, enc(pt, ct, n), seed=bytes(range(32)), scalar=scalar)
    db = processed(entries, res.params)
    assert np.array_equal(res.database.export().astype(np.uint64), db)
    p = osp.ntt_friendly_mod(ct, n)
    assert np.array_equal(res.hint.astype(np.uint64), osp.hint(db, res.params.seed, n, p))
    if size == 600 and count == 40:
        assert res.params.chunksPerEntry > 1 and res.params.aPolyCount > 1


@pytest.mark.parametrize("pt,ct,scalar", [(7, 28, np.uint32), (8, 31, np.uint32), (9, 33, np.uint64), (14, 42, np.uint64),
                                          (16, 61, np.uint64)])
def test_responses_bit_exact_full_width_words(pt, ct, scalar):
    rng = np.random.default_rng(pt * ct)
    prm = sp.SimplePirParameters(enc(pt, ct, 16), 2 * 40, 1, 2, 700)
    db = rng.integers(0, 1 << pt, size=(prm.columnSize, prm.databaseColumns), dtype=np.uint64)
    server = sp.SimplePirServer(db.astype(scalar), np.zeros((prm.columnSize, 16), scalar), prm, scalar)
    info = np.iinfo(scalar)
    reqs = rng.integers(0, int(info.max), size=(9, 2, prm.databaseColumns), dtype=np.uint64, endpoint=True).astype(scalar)
    out = server.computeResponses(reqs)
    for i in range(9):
        assert np.array_equal(out[i].astype(np.uint64), osp.response(db, reqs[i].astype(np.uint64), ct))
        assert np.array_equal(server.computeResponse(reqs[i]), out[i])


def test_all_maximum_operands_cross_every_slice():
    k = 2 * 32768 + 3
    prm = sp.SimplePirParameters(enc(16, 61, 2048), 32, 1, 1, k)  # columnSize 16
    db = np.full((16, k), (1 << 16) - 1, dtype=np.uint64)
    server = sp.SimplePirServer(db, np.zeros((16, 2048), np.uint64), prm)
    req = np.full((3, 1, k), np.iinfo(np.uint64).max, dtype=np.uint64)
    out = server.computeResponses(req)
    expect = ((1 << 16) - 1) * ((1 << 64) - 1) * k % (1 << 61)
    assert np.all(out == np.uint64(expect))
    assert np.array_equal(out[0], osp.response(db, req[0], 61))


def test_one_cta_crosses_every_slice_at_the_bound():
    """4 224 rows and 256 queries fill 4 x 132 CTAs, so K is not split: every CTA runs all three K-slices of
    K = 2 x 32768 + 3 (the first two exactly full at 255 x 255 x 32768) and widens each on its own."""
    k, m = 2 * 32768 + 3, 4224
    prm = sp.SimplePirParameters(enc(16, 31, 2048), 2 * m, 1, 1, k)
    assert prm.columnSize == m
    server = sp.SimplePirServer(np.full((m, k), (1 << 16) - 1, dtype=np.uint32), np.zeros((m, 2048), np.uint32), prm,
                                np.uint32)
    req = np.full((256, 1, k), np.iinfo(np.uint32).max, dtype=np.uint32)
    out = server.computeResponses(req)
    expect = ((1 << 16) - 1) * ((1 << 32) - 1) * k % (1 << 31)  # the oracle's product of any row and any query
    assert np.all(out == np.uint32(expect))
    row = np.full((1, k), (1 << 16) - 1, dtype=np.uint64)
    assert int(osp.response(row, req[0].astype(np.uint64), 31)[0, 0]) == expect


def test_response_crosses_the_grid_y_split():
    """Query-tile pairs go in grid y: 65535 x 16 + 17 queries need a second launch, whose tiles start after the first's."""
    k = 24
    prm = sp.SimplePirParameters(enc(16, 61, 16), 2 * 16, 1, 1, k)
    rng = np.random.default_rng(11)
    db = rng.integers(0, 1 << 16, size=(16, k), dtype=np.uint64)
    server = sp.SimplePirServer(db, np.zeros((16, 16), np.uint64), prm)
    count = 65535 * 16 + 17
    reqs = rng.integers(0, 1 << 63, size=(count, 1, k), dtype=np.uint64)
    server.computeResponses(reqs[:1])
    before = hecuda.kernel_launch_count()
    server.computeResponses(reqs[:1])
    one = hecuda.kernel_launch_count() - before
    before = hecuda.kernel_launch_count()
    out = server.computeResponses(reqs)
    assert hecuda.kernel_launch_count() - before == one + 1
    for i in (0, 65535 * 16 - 1, 65535 * 16, 65535 * 16 + 1, count - 1):
        assert np.array_equal(out[i], osp.response(db, reqs[i], 61)), i


def test_hint_crosses_the_grid_z_split():
    """The hint's inner product puts rows in grid z: 65 540 rows (N = 8, one A polynomial) cross its 65535 split."""
    import ctypes as C

    lib = hecuda.load_library()
    m, k, n = 65540, 3, 8
    prm = sp.SimplePirParameters(enc(8, 9, n), m, 1, 1, k, bytes(range(32)))
    rng = np.random.default_rng(12)
    entries = rng.integers(0, 256, size=(k, m), dtype=np.uint8)
    hint = np.zeros((m, n), dtype=np.uint32)
    seed = np.frombuffer(prm.seed, dtype=np.uint8).copy()
    h = C.c_void_p()
    cp = prm._c(32)
    assert lib.hecuda_simple_pir_process(entries.ctypes.data, k, C.byref(cp), seed.ctypes.data, hint.ctypes.data,
                                         C.byref(h)) == 0
    db = sp.SimplePirDatabase(h, prm, np.uint32)
    expect_db = osp.process_database(entries, 8, 1, 1, k)
    assert np.array_equal(db.export().astype(np.uint64), expect_db)
    assert np.array_equal(hint.astype(np.uint64), osp.hint(expect_db, prm.seed, n, osp.ntt_friendly_mod(9, n)))


def test_device_variant_matches_host_in_stream_order_and_graph_capture():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(5)
    prm = sp.SimplePirParameters(enc(14, 42, 16), 2 * 50, 1, 3, 500)
    db = rng.integers(0, 1 << 14, size=(prm.columnSize, prm.databaseColumns), dtype=np.uint64)
    server = sp.SimplePirServer(db, np.zeros((prm.columnSize, 16), np.uint64), prm)
    reqs = rng.integers(0, 1 << 63, size=(17, 3, 500), dtype=np.uint64)
    host = server.computeResponses(reqs)
    d_req = torch.from_numpy(reqs.view(np.int64)).cuda()
    d_out = torch.zeros((17, 3, prm.columnSize), dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        server.computeResponsesDevice(d_req.data_ptr(), 17, d_out.data_ptr(), s.cuda_stream)
        got = d_out.clone()  # stream order: the clone runs after the response
    s.synchronize()
    assert np.array_equal(got.cpu().numpy().view(np.uint64), host)
    d_out.zero_()
    before = hecuda.kernel_launch_count()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        server.computeResponsesDevice(d_req.data_ptr(), 17, d_out.data_ptr(), s.cuda_stream)
    launched = hecuda.kernel_launch_count() - before
    assert launched > 0
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64), host)


ROUND_TRIPS = [(7, 28, 600, 20, np.uint32), (14, 42, 600, 20, np.uint64), (7, 28, 20, 600, np.uint32),
               (14, 42, 20, 600, np.uint64)]


@pytest.mark.parametrize("pt,ct,count,size,scalar", ROUND_TRIPS)
def test_reference_round_trip_with_the_oracle_client(pt, ct, count, size, scalar):
    """runEncryptDecryptRoundTripTest (N = 1024, errorStdDev 6.4): the oracle's client builds encrypted queries from
    the device's hint, the device answers them, the client decrypts 5 random entries."""
    rng = np.random.default_rng(pt * count)
    entries = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
    res = sp.SimplePirServer.process(entries, enc(pt, ct, 1024, 6.4), scalar=scalar)
    prm = res.params
    server = sp.SimplePirServer(res.database, res.hint, prm, scalar)
    client = osp.Client(dict(N=1024, pt=pt, ct=ct, entries_per_column=prm.entriesPerColumn,
                             chunks_per_entry=prm.chunksPerEntry, database_columns=prm.databaseColumns,
                             entry_size=size), res.hint, prm.seed, rng)
    for index in rng.choice(count, 5, replace=False):
        query, results = client.query(int(index))
        response = server.computeResponse(query.astype(scalar))
        assert client.decrypt(response.astype(np.uint64), results, int(index)) == entries[index].tobytes()


@pytest.mark.parametrize("pt,ct,count,size,scalar", ROUND_TRIPS)
def test_end_to_end_noiseless_retrieval(pt, ct, count, size, scalar):
    rng = random.Random(7 * count + pt)
    entries = raw(rng, count, size)
    res = sp.SimplePirServer.process(entries, enc(pt, ct, 16), scalar=scalar)
    prm = res.params
    server = sp.SimplePirServer(res.database, res.hint, prm, scalar)
    loaded = sp.SimplePirServer(processed(entries, prm).astype(scalar), res.hint, prm, scalar)
    indices = rng.sample(range(count), 5)
    reqs = np.stack([osp.selection_request(i, pt, ct, prm.entriesPerColumn, prm.chunksPerEntry, prm.databaseColumns)
                     for i in indices]).astype(scalar)
    out = server.computeResponses(reqs)
    assert np.array_equal(loaded.computeResponses(reqs), out)
    for i, index in enumerate(indices):
        got = osp.decode_noiseless(out[i].astype(np.uint64), index, pt, ct, size, prm.entriesPerColumn, prm.chunksPerEntry)
        assert got == entries[index].tobytes()


def test_save_load_round_trip_and_truncation(tmp_path):
    rng = random.Random(3)
    entries = raw(rng, 50, 30)
    res = sp.SimplePirServer.process(entries, enc(14, 42, 16))
    path = str(tmp_path / "db.bin")
    res.database.save(path)
    again = sp.SimplePirDatabase.load(path, res.params)
    assert np.array_equal(again.export(), res.database.export())
    sp.save_array2d(res.hint, str(tmp_path / "hint.bin"))
    assert np.array_equal(sp.load_array2d(str(tmp_path / "hint.bin")), res.hint)
    data = open(path, "rb").read()
    open(path, "wb").write(data[:-3])
    with pytest.raises(PirError):
        sp.SimplePirDatabase.load(path, res.params)


def test_refusals_launch_nothing():
    lib = hecuda.load_library()
    before = hecuda.kernel_launch_count()
    good = sp.SimplePirParameters(enc(14, 42, 16), 20, 1, 1, 30)
    entries = np.zeros((30, 20), dtype=np.uint8)
    seed = np.zeros(32, dtype=np.uint8)
    hint = np.zeros((good.columnSize, 16), dtype=np.uint64)
    import ctypes as C

    def process(prm):
        h = C.c_void_p()
        cp = prm._c(64) if isinstance(prm, sp.SimplePirParameters) else prm
        return lib.hecuda_simple_pir_process(entries.ctypes.data, 30, C.byref(cp), seed.ctypes.data, hint.ctypes.data,
                                             C.byref(h))

    bad_n = good._c(64)
    bad_n.lattice_dimension = 24
    assert process(bad_n) == -1
    bad_ct = good._c(64)
    bad_ct.ciphertext_modulus_bits = 14
    assert process(bad_ct) == -1
    wide32 = good._c(32)
    wide32.ciphertext_modulus_bits = 32  # ct + 1 above the UInt32 width
    assert process(wide32) == -2
    wide64 = good._c(64)
    wide64.ciphertext_modulus_bits = 62
    assert process(wide64) == -2
    h = C.c_void_p()
    assert lib.hecuda_simple_pir_process(None, 30, C.byref(good._c(64)), seed.ctypes.data, hint.ctypes.data, C.byref(h)) == -1
    too_big = np.zeros((good.columnSize, 30), dtype=np.uint64)
    too_big[3, 4] = 1 << 14
    with pytest.raises(hecuda.HeError):
        sp.SimplePirDatabase.create(too_big, good)
    assert hecuda.kernel_launch_count() == before
    server = sp.SimplePirServer(np.zeros((good.columnSize, 30), np.uint64), hint, good)
    before = hecuda.kernel_launch_count()
    with pytest.raises(PirError):
        server.computeResponse(np.zeros((1, 29), np.uint64))
    assert lib.hecuda_simple_pir_compute_response(server.database._h, None, 1, hint.ctypes.data) == -1
    assert lib.hecuda_simple_pir_compute_response(server.database._h, hint.ctypes.data, -1, hint.ctypes.data) == -1
    assert hecuda.kernel_launch_count() == before
    with pytest.raises(PirError):
        sp.SimplePirEncryptionParams(14, 43, 2048, 6.4)  # above the quantum128 bound
    sp.SimplePirEncryptionParams(14, 42, 2048, 6.4)
