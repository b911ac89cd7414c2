"""Evaluation keys from the wire (hecuda_evk_create_serialized) and many clients' serialized MulPir queries in one call
(hecuda_mulpir_compute_response_clients_wire).  Loaded keys must be bit-identical to the oracle's expansion of the
seeded key ciphertexts and switch exactly like the same keys uploaded as words; every client's reply bytes must equal
the single-client wire call and the packed oracle composition, and decrypt to the client's database entry."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import evk_wire_ref as ref
import hecuda
from hecuda import pir
from oracle import oracle as orc
from oracle import pir_oracle as opir
from rlwe_shapes import read_device
from test_gpu_pir_clients import CONFIGS, GROUP, Setup

TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)
PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:357-367)
ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, ERR_MISSING_KEY = -1, -2, -5  # HECUDA_ERR_*


def seeded_keys(o, key_seed, rng, elements, galois_seed):
    """A client's secret key and its re-seeded oracle keys: (sk, relin, relin wire (poly0, seeds), {e: key},
    {e: (poly0, seeds)})."""
    sk, relin = o.keygen(key_seed)
    seeds = ref.random_seeds(rng, o.L)
    relin2, relin_poly0 = ref.reseed_key(o, sk, relin, seeds)
    keys, wire = {}, {}
    for i, e in enumerate(elements):
        gseeds = ref.random_seeds(rng, o.L)
        keys[e], poly0 = ref.reseed_key(o, sk, o.galois_keygen(galois_seed + i, sk, e), gseeds)
        wire[e] = (poly0, gseeds)
    return sk, relin2, (relin_poly0, seeds), keys, wire


# ---------------------------------------------------------------- 1. bit-exact keys
KEY_SETS = [
    (16, TEST_MODULI_BITS, 1153, 64),
    (4096, [27, 28, 28], 17, 64),
    (8192, [55, 55, 55, 55], 65537, 64),
    (2048, [62, 62, 62], 65537, 64),
    (4096, PIR_MODULI, 17, 32),
]


@pytest.mark.parametrize("n,bits,t,word_bits", KEY_SETS)
def test_keys_match_oracle_and_switch_like_word_keys(n, bits, t, word_bits):
    moduli = PIR_MODULI if word_bits == 32 else orc.generate_primes(bits, False, n)
    o = orc.Context(n, moduli, t, word_bits=word_bits)
    g = hecuda.Context(n, moduli, t, scalar=np.uint32 if word_bits == 32 else np.uint64)
    rng = np.random.default_rng(n + word_bits)
    elements = [3, 2 * n - 1]
    _, relin, relin_wire, okeys, galois_wire = seeded_keys(o, 21, rng, elements, 40)
    before = hecuda.kernel_launch_count()
    key = hecuda.EvaluationKey.fromSerialized(g, relin_wire[0], relin_wire[1], galois_wire)
    assert hecuda.kernel_launch_count() - before == 2  # one DRBG chain pass, one fused expansion
    assert sorted(key.galoisElements) == elements
    shape = (o.L, 2, o.L + 1, n)
    # expansion of the wire bytes == the re-seeded oracle keys
    for i in range(o.L):
        assert np.array_equal(ref.expand_seeded_key_ciphertext(o, relin_wire[0][i].tobytes(), relin_wire[1][i].tobytes()),
                              relin[i])
    ptr, nbytes = key.deviceBuffer()
    assert nbytes == relin.size * 8
    assert np.array_equal(read_device(ptr, nbytes).reshape(shape), relin)
    for e in elements:
        ptr, nbytes = key.galoisDeviceBuffer(e)
        assert np.array_equal(read_device(ptr, nbytes).reshape(shape), okeys[e]), e
    # relinearize / applyGalois with the wire key == with the same key uploaded as words
    L = o.L
    ct3 = orc.fill_uniform(5, moduli[:L], n, 2 * 3 * L).reshape(2, 3, L, n)
    ct = orc.fill_uniform(6, moduli[:L], n, 2 * 2 * L).reshape(2, 2, L, n)
    if word_bits == 32:
        words = hecuda.EvaluationKey32(g, relin.astype(np.uint32))
        for e in elements:
            words.setGaloisKey(e, okeys[e].astype(np.uint32))
        got = hecuda.Bfv32.relinearize(g, ct3.astype(np.uint32), key)
        assert np.array_equal(got, hecuda.Bfv32.relinearize(g, ct3.astype(np.uint32), words))
        assert np.array_equal(got.astype(np.uint64), o.relinearize(ct3, relin))
        for e in elements:
            assert np.array_equal(hecuda.Bfv32.applyGalois(g, ct.astype(np.uint32), e, key),
                                  hecuda.Bfv32.applyGalois(g, ct.astype(np.uint32), e, words))
    else:
        words = hecuda.EvaluationKey(g, relin)
        for e in elements:
            words.setGaloisKey(e, okeys[e])
        got = hecuda.Bfv.relinearize(g, ct3, key)
        assert np.array_equal(got, hecuda.Bfv.relinearize(g, ct3, words))
        assert np.array_equal(got, o.relinearize(ct3, relin))
        for e in elements:
            assert np.array_equal(hecuda.Bfv.applyGalois(g, ct, e, key), hecuda.Bfv.applyGalois(g, ct, e, words))
    words.close()
    key.close()
    # a key without a relinearization key, and one with nothing at all
    galois_only = hecuda.EvaluationKey.fromSerialized(g, galois={elements[0]: galois_wire[elements[0]]})
    ptr, nbytes = galois_only.galoisDeviceBuffer(elements[0])
    assert np.array_equal(read_device(ptr, nbytes).reshape(shape), okeys[elements[0]])
    with pytest.raises(hecuda.HeError) as err:
        hecuda.Bfv.relinearize(g, ct3, galois_only)
    assert err.value.code == ERR_MISSING_KEY
    galois_only.close()
    hecuda.EvaluationKey.fromSerialized(g).close()
    g.close()


# ---------------------------------------------------------------- 2. everything from the wire
def wire_client(s, seed, rng):
    """A client with its own secret key, a wire-loaded evaluation key and a seeded query."""
    o = s.o
    elements = s.param.evaluationKeyConfig.galoisElements
    sk, relin, relin_wire, okeys, galois_wire = seeded_keys(o, seed, rng, elements, 7000 + 31 * seed)
    key = hecuda.EvaluationKey.fromSerialized(s.g, relin_wire[0], relin_wire[1], galois_wire)
    indices = [s.rng.randrange(s.entries)]
    query = np.stack(opir.generate_query(o, s.oparam, indices, sk, 9000 + seed))
    seeds = ref.random_seeds(rng, len(query))
    cts, poly0 = ref.reseed_query(o, sk, query, seeds)
    return dict(sk=sk, relin=relin, okeys=okeys, key=key, indices=indices, cts=cts, poly0=poly0, seeds=seeds)


def check_wire(s, clients, oracle_clients=None):
    o, n, q0 = s.o, s.o.n, s.o.q[:1]
    replies, skips = pir.PirWire.computeResponses(s.server, np.stack([c["poly0"] for c in clients]),
                                                  np.stack([c["seeds"] for c in clients]), [c["key"] for c in clients])
    assert skips == opir.skip_lsbs_for_decryption(n, q0[0], o.t)
    chunks = s.server.chunkCount
    half = opir.serialization_byte_count(n, q0, skips[0])
    assert replies.shape == (len(clients), 1, chunks, half + opir.serialization_byte_count(n, q0, skips[1]))
    for j, c in enumerate(clients):
        single, _ = pir.PirWire.computeResponse(s.server, c["poly0"], c["seeds"], c["key"])
        assert np.array_equal(replies[j], single), f"client {j} differs from the single-client wire call"
        if oracle_clients is None or j in oracle_clients:
            expected = opir.compute_response(o, list(c["cts"]), 1, c["okeys"], c["relin"], s.odbs, s.oparam)
            for chunk in range(chunks):
                ct = expected[0][chunk]
                want = opir.serialize_poly(n, q0, ct[0], skips[0]) + opir.serialize_poly(n, q0, ct[1], skips[1])
                assert replies[j, 0, chunk].tobytes() == want, (j, chunk)
        recovered = [np.stack([opir.load_poly(n, q0, replies[j, 0, chunk, :half].tobytes(), skips[0]),
                               opir.load_poly(n, q0, replies[j, 0, chunk, half:].tobytes(), skips[1])])
                     for chunk in range(chunks)]
        assert opir.decrypt_response(o, s.oparam, [recovered], c["indices"], c["sk"]) == [s.dbs[0][c["indices"][0]]], j


def contexts(n, bits, t):
    moduli = orc.generate_primes(bits, False, n)
    return hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)


@pytest.mark.parametrize("cfg", CONFIGS)
def test_wire_clients_configs(cfg):
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 100, cfg["entry_size"], cfg["dims"], 1, cfg["uneven"], cfg["compression"], seed=cfg["entry_size"] + 7)
    rng = np.random.default_rng(cfg["entry_size"] * 3 + cfg["dims"])
    clients = [wire_client(s, 40 + c, rng) for c in range(3)]
    check_wire(s, clients)
    s.close(clients)
    g.close()


@pytest.mark.parametrize("count", [1, 2, GROUP, GROUP + 1])
def test_wire_client_counts(count):
    g, o = contexts(16, TEST_MODULI_BITS, 1153)
    s = Setup(g, o, 100, 47, 2, 1, True, "hybridCompression", seed=count)
    rng = np.random.default_rng(count)
    clients = [wire_client(s, 100 + c, rng) for c in range(count)]
    check_wire(s, clients)
    s.close(clients)
    g.close()


def test_wire_clients_pir_parameters():
    g, o = contexts(4096, [27, 28, 28], 17)
    s = Setup(g, o, 20000, 1, 2, 1, True, "hybridCompression", seed=4096)
    rng = np.random.default_rng(4096)
    clients = [wire_client(s, 300 + c, rng) for c in range(2)]
    check_wire(s, clients)
    s.close(clients)
    g.close()


# ---------------------------------------------------------------- 3. errors (all found on the host, before any launch)
def raw_create(g, relin_poly0, relin_seeds, elements, count, galois_poly0, galois_seeds):
    h = C.c_void_p(1)  # not NULL on entry: a failed call must leave NULL behind

    def ptr(a):
        return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)

    rc = hecuda.load_library().hecuda_evk_create_serialized(g._h, ptr(relin_poly0), ptr(relin_seeds), ptr(elements), count,
                                                            ptr(galois_poly0), ptr(galois_seeds), C.byref(h))
    return rc, h


def test_errors():
    n = 16
    g, o = contexts(n, TEST_MODULI_BITS, 1153)
    rng = np.random.default_rng(1)
    _, _, (rp, rs), _, gw = seeded_keys(o, 9, rng, [3], 50)
    gp, gs = gw[3]
    launches = hecuda.kernel_launch_count()
    for args in [
        (rp, None, None, 0, None, None),                             # one of the relinearization arrays missing
        (None, rs, None, 0, None, None),
        (rp, rs, np.array([3], np.uint32), -1, gp, gs),              # negative element_count
        (rp, rs, None, 1, gp, gs),                                   # element_count > 0 with null arrays
        (rp, rs, np.array([3], np.uint32), 1, None, gs),
        (rp, rs, np.array([3], np.uint32), 1, gp, None),
        (rp, rs, np.array([4], np.uint32), 1, gp, gs),               # invalid Galois elements
        (rp, rs, np.array([1], np.uint32), 1, gp, gs),
        (rp, rs, np.array([2 * n + 1], np.uint32), 1, gp, gs),
        (rp, rs, np.array([3, 3], np.uint32), 2, np.concatenate([gp, gp]), np.concatenate([gs, gs])),  # repeated
    ]:
        rc, h = raw_create(g, *args)
        assert rc == ERR_INVALID_ARGUMENT and h.value is None, args[3]
    assert hecuda.kernel_launch_count() == launches
    # a single coefficient modulus has no key-switching modulus
    single = hecuda.Context(n, orc.generate_primes([55], False, n), 1153)
    rc, h = raw_create(single, None, None, None, 0, None, None)
    assert rc == ERR_UNSUPPORTED and h.value is None
    single.close()
    # Python: buffer sizes
    with pytest.raises(hecuda.HeError) as err:
        hecuda.EvaluationKey.fromSerialized(g, rp[:, :-1], rs)
    assert "serializedBufferSizeMismatch" in str(err.value)
    with pytest.raises(hecuda.HeError) as err:
        hecuda.EvaluationKey.fromSerialized(g, rp, rs, {3: (gp, gs[:1])})
    assert "serializedBufferSizeMismatch" in str(err.value)
    with pytest.raises(hecuda.HeError):
        hecuda.EvaluationKey.fromSerialized(g, rp, None)
    # the many-clients wire call checks like the calls it combines
    s = Setup(g, o, 40, 4, 2, 1, False, "noCompression", seed=77)
    clients = [wire_client(s, 500 + c, rng) for c in range(2)]
    poly0 = np.stack([c["poly0"] for c in clients])
    seeds = np.stack([c["seeds"] for c in clients])
    with pytest.raises(hecuda.HeError) as err:
        pir.PirWire.computeResponses(s.server, poly0[:, :, :-1], seeds, [c["key"] for c in clients])
    assert "serializedBufferSizeMismatch" in str(err.value)
    chunks, dims = s.server.chunkCount, s.param.dimensions

    def raw(keys, seeds_arg, skip0=0):
        out = np.empty(4096, dtype=np.uint8)
        handles = (C.c_void_p * 1)(s.server.databases[0]._h)
        key_handles = (C.c_void_p * len(keys))(*[k._h if k is not None else None for k in keys])
        return hecuda.load_library().hecuda_mulpir_compute_response_clients_wire(
            g._h, key_handles, len(keys), handles, 1, (C.c_int32 * len(dims))(*dims), len(dims), chunks,
            poly0.ctypes.data_as(C.c_void_p), None if seeds_arg is None else seeds_arg.ctypes.data_as(C.c_void_p),
            poly0.shape[1], 1, skip0, 0, out.ctypes.data_as(C.c_void_p))

    keys = [c["key"] for c in clients]
    assert raw(keys, None) == ERR_INVALID_ARGUMENT
    assert raw([keys[0], None], seeds) == ERR_MISSING_KEY
    assert "client 1" in hecuda.load_library().hecuda_last_error().decode()
    assert raw(keys, seeds, skip0=64) == ERR_INVALID_ARGUMENT
    assert raw([], seeds) == ERR_INVALID_ARGUMENT
    s.close(clients)
    g.close()


# ---------------------------------------------------------------- 4. concurrent loads
def test_concurrent_loads_are_identical():
    n = 4096
    g, o = contexts(n, [27, 28, 28], 17)
    rng = np.random.default_rng(7)
    elements = [3, 5, 2 * n - 1]
    _, relin, relin_wire, okeys, galois_wire = seeded_keys(o, 12, rng, elements, 60)
    shape = (o.L, 2, o.L + 1, n)
    results, errors = [], []

    def worker():
        try:
            for _ in range(3):
                key = hecuda.EvaluationKey.fromSerialized(g, relin_wire[0], relin_wire[1], galois_wire)
                got = [read_device(*key.deviceBuffer()).reshape(shape)]
                got += [read_device(*key.galoisDeviceBuffer(e)).reshape(shape) for e in elements]
                results.append(got)
                key.close()
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=worker) for _ in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert len(results) == 12
    want = [relin] + [okeys[e] for e in elements]
    for got in results:
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
    g.close()
