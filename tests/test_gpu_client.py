"""The client side of BFV on the GPU: secret keys, encryption (full and seeded), evaluation keys and noise budgets, each
bit-exact (budgets float-exact) against oracle/client_oracle.py for the same seeds; generated keys in use; and PIR
database validation end to end with no oracle involved."""
import ctypes as C
import math
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import keyword_pir as kw
from hecuda import pir, pnns
from oracle import client_oracle as co
from oracle import oracle as orc
from oracle import pir_oracle as opir
from rlwe_shapes import read_device, seed

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]  # bench.py C2 moduli
T_C2 = 557057
PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28 (EncryptionParameters.swift:346-367)
PARAMS = [(4096, Q8192, T_C2), (8192, Q8192, T_C2), (4096, PIR_MODULI, 17)]
IDS = ["n4096-c2", "n8192-c2", "n4096-pir"]


@pytest.fixture(scope="module", params=PARAMS, ids=IDS)
def setup(request):
    n, moduli, t = request.param
    g = hecuda.Context(n, moduli, t)
    sk = hecuda.SecretKey.generate(g, seed(1))
    yield n, moduli, t, g, sk
    g.close()


def _plaintexts(n, t, count, rs):
    rng = np.random.default_rng(rs)
    return rng.integers(0, t, size=(count, n), dtype=np.uint64)


def test_secret_key_matches_oracle(setup):
    n, moduli, t, g, sk = setup
    assert np.array_equal(sk.poly, co.generate_secret_key(n, moduli, seed(1)))
    seeds = np.frombuffer(seed(2) + seed(3) + seed(4), dtype=np.uint8).reshape(3, 32).copy()
    out = np.empty((3, len(moduli), n), dtype=np.uint64)
    assert hecuda.load_library().hecuda_bfv_generate_secret_key(g._h, hecuda._ptr(seeds), hecuda._ptr(out), 3) == 0
    for i in range(3):
        assert np.array_equal(out[i], co.generate_secret_key(n, moduli, bytes(seeds[i])))


def test_encrypt_matches_oracle_and_decrypts(setup):
    n, moduli, t, g, sk = setup
    L = g.L
    pts = _plaintexts(n, t, 3, 5)
    a = [seed(10 + i) for i in range(3)]
    e = [seed(20 + i) for i in range(3)]
    cts = hecuda.Bfv.encrypt(g, sk, pts, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    assert cts.shape == (3, 2, L, n)
    for i in range(3):
        assert np.array_equal(cts[i], co.encrypt(n, moduli[:L], t, sk.poly, pts[i], a[i], e[i])), i
    assert np.array_equal(hecuda.Bfv.decrypt(g, cts, sk), pts)
    fresh = hecuda.Bfv.encrypt(g, sk, pts)  # seeds from secrets.token_bytes
    assert np.array_equal(hecuda.Bfv.decrypt(g, fresh, sk), pts)
    assert not np.array_equal(fresh, cts)


def test_seeded_wire_form_expands_to_the_full_ciphertext(setup):
    n, moduli, t, g, sk = setup
    L = g.L
    pts = _plaintexts(n, t, 2, 6)
    a, e = seed(30) + seed(31), seed(40) + seed(41)
    full = hecuda.Bfv.encrypt(g, sk, pts, aSeeds=a, errorSeeds=e)
    poly0, seeds = hecuda.Bfv.encrypt(g, sk, pts, seeded=True, aSeeds=a, errorSeeds=e)
    assert np.array_equal(seeds.reshape(-1), np.frombuffer(a, dtype=np.uint8))
    for i in range(2):
        assert bytes(poly0[i]) == opir.serialize_poly(n, moduli[:L], full[i, 0])
    assert np.array_equal(hecuda.Bfv.expandSeeded(g, poly0, seeds), full)


def _config(n):
    return pir.EvaluationKeyConfig([3, 2 * n - 1], True)


def test_evaluation_key_matches_oracle_and_its_wire_form(setup):
    n, moduli, t, g, sk = setup
    L = g.L
    count = 3 * L
    a = [seed(100 + i) for i in range(count)]
    e = [seed(200 + i) for i in range(count)]
    key, form = hecuda.EvaluationKey.generate(g, _config(n), sk, wire=True, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    relin, galois = co.generate_evaluation_key(n, moduli[:L], moduli[L], sk.poly, True, [3, 2 * n - 1], a, e)
    assert np.array_equal(read_device(*key.deviceBuffer()).reshape(relin.shape), relin)
    for el in (3, 2 * n - 1):
        assert np.array_equal(read_device(*key.galoisDeviceBuffer(el)).reshape(relin.shape), galois[el]), el
    loaded = hecuda.EvaluationKey.fromSerialized(g, **form)
    assert np.array_equal(read_device(*loaded.deviceBuffer()), read_device(*key.deviceBuffer()))
    for el in (3, 2 * n - 1):
        assert np.array_equal(read_device(*loaded.galoisDeviceBuffer(el)), read_device(*key.galoisDeviceBuffer(el)))
    loaded.close()
    key.close()


def test_generated_keys_in_use(setup):
    n, moduli, t, g, sk = setup
    L = g.L
    o = orc.Context(n, moduli, t)
    count = 3 * L
    a, e = [seed(300 + i) for i in range(count)], [seed(400 + i) for i in range(count)]
    key = hecuda.EvaluationKey.generate(g, _config(n), sk, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    relin, galois = co.generate_evaluation_key(n, moduli[:L], moduli[L], sk.poly, True, [3, 2 * n - 1], a, e)
    pts = _plaintexts(n, t, 2, 7)
    cts = hecuda.Bfv.encrypt(g, sk, pts)
    prod = hecuda.Bfv.mulAssign(g, cts[:1], cts[1:])
    relinearized = hecuda.Bfv.relinearize(g, prod, key)
    assert np.array_equal(relinearized[0], o.relinearize(prod, relin)[0])
    assert np.array_equal(hecuda.Bfv.decrypt(g, relinearized, sk), hecuda.Bfv.decrypt(g, prod, sk))
    assert np.array_equal(hecuda.Bfv.decrypt(g, relinearized, sk)[0], o.decrypt(sk.poly, o.mul(cts[:1], cts[1:])[0]))
    for el in (3, 2 * n - 1):
        rotated = hecuda.Bfv.applyGalois(g, cts, el, key)
        assert np.array_equal(rotated, o.apply_galois(cts, el, galois[el]))
        expected = np.stack([orc.galois_coeff(n, [t], el, p[None])[0] for p in pts])
        assert np.array_equal(hecuda.Bfv.decrypt(g, rotated, sk), expected)
    key.close()


def _budgets_match(g, n, moduli, t, sk, cts, eval_format=False):
    got = hecuda.Bfv.noiseBudget(g, sk, cts, evalFormat=eval_format)
    for i, ct in enumerate(cts):
        assert got[i] == co.noise_budget(n, moduli, t, sk.poly, ct, eval_format), i
    return got


def test_noise_budget_matches_oracle(setup):
    n, moduli, t, g, sk = setup
    L = g.L
    pts = _plaintexts(n, t, 2, 8)
    cts = hecuda.Bfv.encrypt(g, sk, pts)
    fresh = _budgets_match(g, n, moduli, t, sk, cts)
    assert np.all(fresh > 0)
    ev = np.stack([np.stack([orc.ntt_forward(n, moduli[:L], ct[p]) for p in range(2)]) for ct in cts])
    assert np.array_equal(_budgets_match(g, n, moduli, t, sk, ev, eval_format=True), fresh)
    key = hecuda.EvaluationKey.generate(g, pir.EvaluationKeyConfig([], True), sk)
    product = hecuda.Bfv.mulRelinearize(g, cts[:1], cts[1:], key)
    budget = _budgets_match(g, n, moduli, t, sk, product)
    assert budget[0] < fresh.min()
    if L >= 2:
        _budgets_match(g, n, moduli, t, sk, hecuda.Bfv.modSwitchDown(g, product))
    three = hecuda.Bfv.mulAssign(g, cts[:1], cts[1:])
    _budgets_match(g, n, moduli, t, sk, three)
    zero = np.zeros((1, 2, L, n), dtype=np.uint64)
    assert hecuda.Bfv.noiseBudget(g, sk, zero)[0] == math.inf
    assert hecuda.Bfv.noiseBudget(g, sk, zero[0], evalFormat=True) == math.inf
    key.close()


@pytest.fixture(scope="module")
def pir_context():
    g = hecuda.Context(4096, PIR_MODULI, 17)
    yield g
    g.close()


def _index_server(g, entries, dims=2):
    config = pir.IndexPirConfig(len(entries), max(len(x) for x in entries), dims, 1, False, "hybridCompression", True)
    parameter = pir.MulPir.generateParameter(config, g)
    return pir.MulPirServer(parameter, g, [pir.MulPirServer.processOnDevice(entries, g, parameter)])


def test_noise_budget_of_mulpir_and_pnns_replies(pir_context):
    g = pir_context
    rng = random.Random(3)
    entries = [rng.randbytes(rng.randrange(1, 40)) for _ in range(300)]
    server = _index_server(g, entries)
    client = pir.MulPirClient(server.parameter, g)
    sk = hecuda.SecretKey.generate(g)
    key = client.generateEvaluationKey(sk)
    response = server.computeResponse(client.generateQuery([123], sk), key)
    assert client.decrypt(response, [123], sk) == [entries[123]]
    replies = response.reshape(-1, 2, 1, 4096)
    _budgets_match(g, 4096, PIR_MODULI, 17, sk, replies)
    assert client.noiseBudget(response, sk) == min(co.noise_budget(4096, PIR_MODULI, 17, sk.poly, r) for r in replies)
    key.close()
    # a PNNS reply (M v^T), keys and query from the device client
    n, t, moduli = 4096, 65537, orc.generate_primes([36, 36, 37], False, 4096)
    gp = hecuda.Context(n, moduli, t)
    rows, cols = 50, 16
    matrix = [rng.randrange(t) for _ in range(rows * cols)]
    device_matrix = pnns.PlaintextMatrix(gp, pnns.MatrixDimensions(rows, cols), matrix)
    elements = [pnns.GaloisElement.rotatingColumns(-1, n)]
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(cols)
    if bsgs.giantStep > 1:
        elements.append(pnns.GaloisElement.rotatingColumns(-bsgs.babyStep, n))
    skp = hecuda.SecretKey.generate(gp)
    keyp = hecuda.EvaluationKey.generate(gp, pir.EvaluationKeyConfig(list(dict.fromkeys(elements)), False), skp)
    vector = [rng.randrange(t) for _ in range(cols)]
    ct = hecuda.Bfv.encrypt(gp, skp, np.asarray(pnns.denseRowVector(gp, vector), dtype=np.uint64)[None])
    reply = device_matrix.mulTranspose(ct, keyp, modSwitchDownToSingle=True)
    _budgets_match(gp, n, moduli, t, skp, reply.reshape(-1, 2, reply.shape[-2], n))
    device_matrix.close()
    keyp.close()
    gp.close()


def test_mulpir_validate_end_to_end(pir_context):
    g = pir_context
    rng = random.Random(4)
    entries = [rng.randbytes(rng.randrange(1, 60)) for _ in range(500)]
    server = _index_server(g, entries)
    result = server.validate((77, entries[77]), trials=2)
    assert result.decryptedRow == entries[77]
    assert result.noiseBudget > hecuda.Bfv.minNoiseBudget and math.isfinite(result.noiseBudget)
    assert len(result.computeTimes) == 2 and result.entryCountPerResponse == [1, 1]
    assert result.query.shape[1:] == (2, g.L, 4096)
    result.evaluationKey.close()
    altered = list(entries)
    altered[77] = bytes(b ^ 1 for b in altered[77])
    bad = _index_server(g, altered)
    with pytest.raises(pir.PirError, match="Incorrect PIR response"):
        bad.validate((77, entries[77]), trials=1)
    with pytest.raises(pir.PirError, match="Invalid trialsPerShard"):
        server.validate((77, entries[77]), trials=0)


def test_keyword_validate_end_to_end(pir_context):
    g = pir_context
    rng = random.Random(5)
    rows = [(b"keyword %d" % i, rng.randbytes(rng.randrange(1, 30))) for i in range(300)]
    config = kw.KeywordPirConfig(2, kw.CuckooTableConfig.defaultKeywordPir(200), False, "hybridCompression")
    processed = kw.KeywordPirServer.processOnDevice(rows, config, g)
    server = kw.KeywordPirServer(g, processed)
    result = server.validate(rows[11], trials=2)
    assert result.decryptedRow == rows[11][1]
    assert result.noiseBudget > hecuda.Bfv.minNoiseBudget and math.isfinite(result.noiseBudget)
    assert all(c >= 1 for c in result.entryCountPerResponse)
    result.evaluationKey.close()
    altered = list(rows)
    altered[11] = (rows[11][0], bytes(b ^ 1 for b in rows[11][1]))
    bad = kw.KeywordPirServer(g, kw.KeywordPirServer.processOnDevice(altered, config, g))
    with pytest.raises(pir.PirError, match="Incorrect PIR response"):
        bad.validate(rows[11], trials=1)
    bad.processed.close()
    processed.close()


def test_bad_arguments_launch_nothing(pir_context):
    g = pir_context
    lib = hecuda.load_library()
    n, L = 4096, g.L
    sk = hecuda.SecretKey.generate(g)
    pts = np.zeros((1, n), dtype=np.uint64)
    seeds = np.zeros((3 * L, 32), dtype=np.uint8)
    ct = np.zeros((1, 2, L, n), dtype=np.uint64)
    out = np.empty((1, 2, L, n), dtype=np.uint64)
    budgets = np.empty(1)
    h = C.c_void_p()
    p = hecuda._ptr
    before = hecuda.kernel_launch_count()
    assert lib.hecuda_bfv_encrypt(g._h, None, p(pts), p(seeds), p(seeds), p(out), 1) == -5
    assert lib.hecuda_bfv_encrypt(g._h, p(sk.poly), p(pts), None, p(seeds), p(out), 1) == -1
    assert lib.hecuda_bfv_encrypt(g._h, p(sk.poly), p(pts + 17), p(seeds), p(seeds), p(out), 1) == -1  # value >= t
    assert lib.hecuda_bfv_encrypt_seeded(g._h, p(sk.poly), p(pts), p(seeds), None, p(out), 1) == -1
    assert lib.hecuda_bfv_generate_secret_key(g._h, None, p(out), 1) == -1
    elems = np.array([3], dtype=np.uint32)
    assert lib.hecuda_evk_generate(g._h, None, 1, p(elems), 1, p(seeds), p(seeds), C.byref(h), None) == -5
    assert lib.hecuda_evk_generate(g._h, p(sk.poly), 1, p(elems), 1, None, p(seeds), C.byref(h), None) == -1
    for bad in ([4], [1], [2 * n + 1], [3, 3]):
        el = np.array(bad, dtype=np.uint32)
        assert lib.hecuda_evk_generate(g._h, p(sk.poly), 0, p(el), len(bad), p(seeds), p(seeds), C.byref(h), None) == -1
        assert h.value is None
    assert lib.hecuda_bfv_noise_budget(g._h, None, p(ct), 2, L, 0, p(budgets), 1) == -5
    for l in (0, L + 1):
        assert lib.hecuda_bfv_noise_budget(g._h, p(sk.poly), p(ct), 2, l, 0, p(budgets), 1) == -1
    assert lib.hecuda_bfv_noise_budget(g._h, p(sk.poly), p(ct), 4, L, 0, p(budgets), 1) == -1
    assert lib.hecuda_bfv_noise_budget(g._h, p(sk.poly), None, 2, L, 0, p(budgets), 1) == -1
    assert hecuda.kernel_launch_count() == before
