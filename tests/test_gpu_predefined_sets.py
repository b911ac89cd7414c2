"""The BFV operations at every predefined parameter set of the reference, and at two contexts that mix every NTT class
at N = 2^12 and 2^13, bit-exact against the oracles.

The predefined sets (tests/behz_bounds.py PREDEFINED) are what the reference's users pick: N from 8 to 8192, one to four
ciphertext moduli of 16 to 60 bits, plaintext moduli with and without SIMD.  Each set reaches code that the uniform
shapes of the other files do not: N = 8 and 16 with key switching, one coefficient modulus and so no key switching at
all, MID rows below the fast NTT's smallest degree, a 16-bit q_0 that is the whole last level, SMALL or NARROW q_0 next
to MID rows at N = 8192, and the reference's Bsk instead of the auxiliary base.  The mixed shapes:

  M12-mixed, M13-mixed  N = 2^12 and 2^13, rows of 62, 30, 55, h 2^32 + 1, 31 and 61 bits, a 56-bit key-switching
                        modulus, t = 786433: every class of csrc/ntt_fast.cuh in one context, the 62-bit row first.
                        With one class per context the NTT's class-major row order is the identity, so a row mapped
                        back to the wrong place, or a key-switching modulus of another class reduced with the wrong
                        schedule, is only seen here below N = 2^15.

Each shape asserts the property it was chosen for.  Secret keys, encryptions and evaluation keys (relinearization,
rotate by 1, rotate by -N/4, swap rows) are generated on the device from fixed seeds and compared with the client oracle
over every key ciphertext, and every later test uses those keys.  Besides bit-exact parity, the stages of the multiply
chain and the Galois images are decrypted and compared with the plaintext arithmetic itself: a negacyclic product with
a sparse operand, and m(x^e) mod (x^N + 1).  That is sound while the oracle's noise budget keeps a margin (decrypts_to);
with these seeds the relinearized chain and every Galois image keep it at every level, and the tests assert so.

The seven sets the reference marks supportsScalar32 also run the evaluator through Bfv<UInt32> (`-u32` ids): the NTT,
multiply, relinearize, modSwitchDown, the fused calls, applyGalois and the ct x ct inner product.  The library has no
UInt32 client operations, so those tests use the 64-bit keys, whose residues are the same.

Every key ciphertext is compared: at N <= 8192 the client oracle's Python sampling of all of them takes about 14 s on
one CPU core, 4 s of it for M13-mixed.  The file's 176 tests run in about 50 s on one H100 (80 GB HBM3, 700 W)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

import behz_bounds as bb  # noqa: E402
import hecuda  # noqa: E402
from hecuda import pir  # noqa: E402
from oracle import client_oracle as co  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from oracle import pir_oracle as opir  # noqa: E402
from rlwe_shapes import (MID, NARROW, NARROW_H, SMALL, WIDE, keyed_elements, mixed_moduli, modulus_class,  # noqa: E402
                         read_device, seed)
from test_gpu_behz_bounds import MUL_SETS, check_multiply  # noqa: E402

SETS = list(bb.PREDEFINED)
MIXED = {"M12-mixed": 1 << 12, "M13-mixed": 1 << 13}
SHAPES = SETS + list(MIXED)
T_MIXED = 786433  # 3 * 2^18 + 1, prime, 2^14 | t - 1
SINGLE = "insecure_n_16_logq_60_logt_15"
# supportsScalar32: true (EncryptionParameters.swift)
U32_SETS = ["insecure_n_8_logq_5x18_logt_5"] + [name for name in SETS if "_27_28_28_" in name]
FAST_MIN_LOG_N = 10  # fast::kMinLogN: smaller degrees run the simple NTT
IP_TERMS = [1, 17]
MIN_BUDGET = 0.5  # bits: see decrypts_to
ERR_UNSUPPORTED, ERR_MISSING_KEY = -2, -5  # HECUDA_ERR_*


def shape_params(name):
    """(N, coefficient moduli, t) of a shape."""
    if name in bb.PREDEFINED:
        n, moduli, t, _ = bb.PREDEFINED[name]
        return n, list(moduli), t
    return MIXED[name], mixed_moduli(MIXED[name]), T_MIXED


def assert_chosen_property(s):
    n, classes = s.n, [modulus_class(p) for p in s.moduli]
    if s.name == SINGLE:
        assert len(s.moduli) == 1 and s.L == 1 and not s.has_ks
    elif s.name == "insecure_n_8_logq_5x18_logt_5":
        assert n == 8 and s.L == 4 and set(classes) == {SMALL}
    elif s.name == "insecure_n_512_logq_4x60_logt_20":
        assert n < 1 << FAST_MIN_LOG_N and set(classes) == {MID}
    elif s.name == "n_4096_logq_16_33_33_logt_4":
        assert s.q[0] == 40961 and classes == [SMALL, NARROW, NARROW] and s.t == 11
    elif "_27_28_28_" in s.name:
        assert n == 4096 and set(classes) == {SMALL}
    elif "_60_60_" in s.name:
        assert n == 8192 and classes[0] in (SMALL, NARROW) and classes[1:] == [MID, MID]
    elif "_3x55_" in s.name:
        assert n == 8192 and set(classes) == {NARROW}
    else:
        assert s.name in MIXED
        assert {SMALL, NARROW, NARROW_H, MID, WIDE} <= set(classes)
        assert classes[0] == WIDE and WIDE not in classes[1:]
        assert (s.t - 1) % (2 * n) == 0 and s.g.supportsSimdEncoding
    # the base the multiply computes in: the auxiliary base of 30- or 55-bit primes, or the reference's Bsk
    aux, bsk = bb.aux_base(n, s.moduli, s.t)
    assert s.g.auxModuli == aux and s.g.bskModuli == bsk
    kind = bb.PREDEFINED[s.name][3] if s.name in bb.PREDEFINED else 55
    if kind == "bsk":
        assert aux == bsk
    else:
        assert aux != bsk and max(aux).bit_length() <= kind


class Shape:
    """One shape: device and oracle contexts, a secret key and (with a key-switching modulus) an evaluation key generated
    on the device from fixed seeds, with host copies of the evaluation key."""

    def __init__(self, name):
        self.name = name
        self.n, self.moduli, self.t = shape_params(name)
        n = self.n
        assert all(p % (2 * n) == 1 for p in self.moduli), "NTT-friendly at this N"
        self.g = hecuda.Context(n, self.moduli, self.t)
        self.L, self.q = self.g.L, self.g.ciphertextModuli
        self.has_ks = len(self.moduli) > 1
        # The C oracle's context needs a key-switching modulus.  With one coefficient modulus it gets a spare one, which
        # its ciphertext operations never touch (the multiply's Bsk depends on L alone).
        spare = [] if self.has_ks else [p for p in orc.generate_primes([59] * 2, False, n) if p not in self.moduli][:1]
        self.o = orc.Context(n, self.moduli + spare, self.t)
        assert self.o.L == self.L
        self.elements = list(dict.fromkeys(keyed_elements(n)))
        assert len(self.elements) == 3
        self.sk = hecuda.SecretKey.generate(self.g, seed(1))
        self.evk = None
        if self.has_ks:
            count = (1 + len(self.elements)) * self.L
            self.a_seeds = [seed(1000 + i) for i in range(count)]
            self.e_seeds = [seed(2000 + i) for i in range(count)]
            self.evk, self.wire = hecuda.EvaluationKey.generate(
                self.g, pir.EvaluationKeyConfig(self.elements, True), self.sk, wire=True,
                aSeeds=b"".join(self.a_seeds), errorSeeds=b"".join(self.e_seeds))
            key_shape = (self.L, 2, self.L + 1, n)
            self.relin = read_device(*self.evk.deviceBuffer()).reshape(key_shape)
            self.galois = {e: read_device(*self.evk.galoisDeviceBuffer(e)).reshape(key_shape) for e in self.elements}
        assert_chosen_property(self)

    def plaintexts(self, count, rs):
        pts = np.random.default_rng(rs).integers(0, self.t, size=(count, self.n), dtype=np.uint64)
        pts[0, :2] = [0, self.t - 1]
        return pts

    def sparse(self, rs):
        """A plaintext with four nonzero coefficients, at 0, 1, N/2 and N - 1, one of them t - 1."""
        pt = np.zeros(self.n, dtype=np.uint64)
        at = [0, 1, self.n // 2, self.n - 1]
        pt[at] = np.random.default_rng(rs).integers(1, self.t, size=len(at), dtype=np.uint64)
        pt[self.n // 2] = self.t - 1
        return pt

    def encrypt(self, pts, first_seed):
        """Device encryptions of (count, N) plaintexts with the seeds first_seed, first_seed + 1, ..."""
        a = [seed(first_seed + i) for i in range(len(pts))]
        e = [seed(first_seed + 500 + i) for i in range(len(pts))]
        return hecuda.Bfv.encrypt(self.g, self.sk, pts, aSeeds=b"".join(a), errorSeeds=b"".join(e))

    def budget(self, ct):
        return co.noise_budget(self.n, self.moduli, self.t, self.sk.poly, ct)

    def close(self):
        if self.evk is not None:
            self.evk.close()
        self.g.close()


@pytest.fixture(scope="module")
def shapes():
    built = {}

    def get(name):
        if name not in built:
            built[name] = Shape(name)
        return built[name]

    yield get
    for s in built.values():
        s.close()


def negacyclic_times_sparse(m, sparse, t):
    """m * sparse mod (x^N + 1, t), summing one signed shift of m per nonzero coefficient of `sparse`."""
    n = len(m)
    m = m.astype(object)
    out = np.zeros(n, dtype=object)
    for j in np.flatnonzero(sparse):
        out += int(sparse[j]) * np.concatenate([-m[n - j:], m[:n - j]])
    return (out % t).astype(np.uint64)


def decrypts_to(s, ct, want):
    """Whether the device decryption of the (polys, l, N) ciphertext was compared with `want`: it is when the oracle's
    noise budget is at least MIN_BUDGET.

    A positive budget alone does not do: the noise norm is the largest centred [t v]_q, which is below q/2 by
    construction.  When the noise has wrapped, those values are close to uniform and their maximum over N
    coefficients is about q/2 (1 - 1/N), a budget of about 1 / (N ln 2) bits -- the three-polynomial product switched
    down to one 28-bit modulus shows 0.0001 bits and decrypts to other values.  N wrapped coefficients all stay below
    q / 2^1.5 with probability 2^(-N/2)."""
    if s.budget(ct) < MIN_BUDGET:
        return False
    assert np.array_equal(hecuda.Bfv.decrypt(s.g, ct[None], s.sk)[0], want), ct.shape
    return True


# ------------------------------------------------------------------------------------------------------------ client
@pytest.mark.parametrize("name", SHAPES)
def test_secret_key_and_encryption_match_client_oracle(shapes, name):
    s = shapes(name)
    n, q = s.n, s.q
    assert np.array_equal(s.sk.poly, co.generate_secret_key(n, s.moduli, seed(1)))
    pts = s.plaintexts(2, 5)
    a, e = [seed(10), seed(11)], [seed(20), seed(21)]
    full = hecuda.Bfv.encrypt(s.g, s.sk, pts, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    for i in range(2):
        assert np.array_equal(full[i], co.encrypt(n, q, s.t, s.sk.poly, pts[i], a[i], e[i])), i
    assert np.array_equal(hecuda.Bfv.decrypt(s.g, full, s.sk), pts)
    poly0, seeds = hecuda.Bfv.encrypt(s.g, s.sk, pts, seeded=True, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    assert np.array_equal(seeds.reshape(-1), np.frombuffer(b"".join(a), dtype=np.uint8))
    for i in range(2):
        assert bytes(poly0[i]) == opir.serialize_poly(n, q, full[i, 0]), i
    assert np.array_equal(hecuda.Bfv.expandSeeded(s.g, poly0, seeds), full)


@pytest.mark.parametrize("name", SHAPES)
def test_evaluation_key_matches_client_oracle(shapes, name):
    """Every key ciphertext of the relinearization key and of the three Galois keys, and the key loaded back from its
    seeded wire form.  With a single coefficient modulus there is no key-switching modulus, so every way of making an
    evaluation key, and relinearizing without one, is refused (Context.swift:102-107)."""
    s = shapes(name)
    if not s.has_ks:
        lib = hecuda.load_library()
        h = C.c_void_p()
        count = (1 + len(s.elements)) * s.L
        elems = np.array(s.elements, dtype=np.uint32)
        a = np.frombuffer(b"".join(seed(1000 + i) for i in range(count)), dtype=np.uint8).copy()
        e = np.frombuffer(b"".join(seed(2000 + i) for i in range(count)), dtype=np.uint8).copy()
        assert lib.hecuda_evk_generate(s.g._h, hecuda._ptr(s.sk.poly), 1, hecuda._ptr(elems), len(elems),
                                       hecuda._ptr(a), hecuda._ptr(e), C.byref(h), None) == ERR_UNSUPPORTED
        assert lib.hecuda_evk_create_empty(s.g._h, C.byref(h)) == ERR_UNSUPPORTED
        assert lib.hecuda_evk_create_serialized(s.g._h, None, None, None, 0, None, None, C.byref(h)) == ERR_UNSUPPORTED
        assert h.value is None
        with pytest.raises(hecuda.HeError):
            hecuda.EvaluationKey(s.g, np.zeros((1, 2, 2, s.n), dtype=np.uint64))
        product = s.o.mul(*s.encrypt(s.plaintexts(2, 6), 50)[:, None])
        out = np.empty((1, 2, 1, s.n), dtype=np.uint64)
        assert lib.hecuda_bfv_relinearize(s.g._h, None, hecuda._ptr(product), 1, hecuda._ptr(out), 1) == ERR_MISSING_KEY
        return
    relin, galois = co.generate_evaluation_key(s.n, s.q, s.moduli[s.L], s.sk.poly, True, s.elements, s.a_seeds,
                                               s.e_seeds)
    assert np.array_equal(s.relin, relin)
    for el in s.elements:
        assert np.array_equal(s.galois[el], galois[el]), el
    loaded = hecuda.EvaluationKey.fromSerialized(s.g, **s.wire)
    assert np.array_equal(read_device(*loaded.deviceBuffer()), s.relin.reshape(-1))
    for el in s.elements:
        assert np.array_equal(read_device(*loaded.galoisDeviceBuffer(el)), s.galois[el].reshape(-1)), el
    loaded.close()


# ------------------------------------------------------------------------------------------------------------ multiply
@pytest.mark.parametrize("name", SHAPES)
def test_multiply_relinearize_and_mod_switch_down(shapes, name):
    """multiply -> relinearize -> modSwitchDown to one modulus (the three-polynomial product too), every stage against
    the oracle and, while its noise budget allows, decrypted to the negacyclic product; the fused calls equal the
    separate ones."""
    s = shapes(name)
    g, o, t = s.g, s.o, s.t
    m, sp = s.plaintexts(1, 3)[0], s.sparse(4)
    cts = s.encrypt(np.stack([m, sp]), 60)
    a, b = cts[:1], cts[1:]
    want = negacyclic_times_sparse(m, sp, t)
    product = hecuda.Bfv.mulAssign(g, a, b)
    assert np.array_equal(product, o.mul(a, b))
    assert decrypts_to(s, product[0], want)
    if not s.has_ks:
        with pytest.raises(hecuda.HeError):  # no next level
            hecuda.Bfv.modSwitchDown(g, product)
        return
    relin = hecuda.Bfv.relinearize(g, product, s.evk)
    assert np.array_equal(relin, o.relinearize(product, s.relin))
    assert decrypts_to(s, relin[0], want)
    assert np.array_equal(hecuda.Bfv.mulRelinearize(g, a, b, s.evk), relin)
    ct, ct3, level = relin, product, s.L
    while level > 1:
        down = hecuda.Bfv.modSwitchDown(g, ct)
        assert np.array_equal(down, o.mod_switch_down(ct)), level
        down3 = hecuda.Bfv.modSwitchDown(g, ct3)
        assert np.array_equal(down3, o.mod_switch_down(ct3)), level
        if level == s.L:
            assert np.array_equal(hecuda.Bfv.mulRelinearize(g, a, b, s.evk, modSwitchDown=True), down)
            assert np.array_equal(hecuda.Bfv.relinearizeModSwitchDown(g, product, s.evk), down)
        assert decrypts_to(s, down[0], want), level
        decrypts_to(s, down3[0], want)  # its noise wraps at the last level of five sets
        ct, ct3, level = down, down3, level - 1
    assert ct.shape[-2] == 1


@pytest.mark.parametrize("name", [name for name in SHAPES if name not in MUL_SETS])
def test_multiply_at_aligned_operands(shapes, name):
    """tests/test_gpu_behz_bounds.py's worst-case multiply at the shapes its MUL_SETS leaves out: the oracle's words,
    and floor(t D / q) within the floor's tolerance on sampled coefficients."""
    s = shapes(name)
    check_multiply(s.g, s.o, s.n, s.q, s.t)


# ------------------------------------------------------------------------------------------------------------ Galois
@pytest.mark.parametrize("name", SHAPES)
def test_apply_galois_with_generated_keys(shapes, name):
    """Bfv.applyGalois with the device-generated keys at every level: the oracle's words, and the encrypted message
    permuted with sign flips, m(x^e).  With a single coefficient modulus there are no keys: the permutation itself."""
    s = shapes(name)
    n, q, L, t = s.n, s.q, s.L, s.t
    m = s.plaintexts(1, 10)[0]
    ct = np.concatenate([s.encrypt(m[None], 70), orc.fill_uniform(71, q, n, 2 * L).reshape(1, 2, L, n)])
    if not s.has_ks:
        for el in s.elements:
            got = hecuda.Bfv.polyApplyGalois(s.g, ct, el)
            for k in range(2):
                for p in range(2):
                    assert np.array_equal(got[k, p], orc.galois_coeff(n, q, el, ct[k, p])), (el, k, p)
        return
    level = L
    while True:
        for el in s.elements:
            got = hecuda.Bfv.applyGalois(s.g, ct, el, s.evk)
            assert np.array_equal(got, s.o.apply_galois(ct, el, s.galois[el])), (el, level)
            assert decrypts_to(s, got[0], orc.galois_coeff(n, [t], el, m[None])[0]), (el, level)
        if level == 1:
            break
        ct, level = s.o.mod_switch_down(ct), level - 1


# ---------------------------------------------------------------------------------------------------- inner products
@pytest.mark.parametrize("terms", IP_TERMS)
@pytest.mark.parametrize("name", SHAPES)
def test_inner_products(shapes, name, terms):
    """ct x pt (plaintexts through plaintextToEval) at the top level and at one modulus, and ct x ct, against the
    oracle, with all-(q_i - 1) coefficients in the first term."""
    s = shapes(name)
    n, q, L, t, o = s.n, s.q, s.L, s.t, s.o
    rows = 2
    ps = np.random.default_rng(terms).integers(0, t, size=(rows * terms, n), dtype=np.uint64)
    ps[0, :2] = [0, t - 1]
    for level in sorted({L, 1}):
        pts = hecuda.Bfv.plaintextToEval(s.g, ps, level)
        assert np.array_equal(pts, np.stack([o.plaintext_to_eval(p, level) for p in ps])), level
        pts = pts.reshape(rows, terms, level, n)
        cts = orc.fill_uniform(terms + level, q[:level], n, terms * 2 * level).reshape(terms, 2, level, n)
        for i, p in enumerate(q[:level]):
            cts[0, :, i, :4] = p - 1
        got = hecuda.Bfv.innerProduct(s.g, cts, pts)
        assert np.array_equal(got, o.inner_product_plain(cts, pts)), level
    lhs = orc.fill_uniform(terms + 20, q, n, terms * 2 * L).reshape(1, terms, 2, L, n)
    rhs = orc.fill_uniform(terms + 30, q, n, terms * 2 * L).reshape(1, terms, 2, L, n)
    for i, p in enumerate(q):
        lhs[0, 0, :, i, :4] = p - 1
        rhs[0, 0, :, i, :4] = [0, 1, p - 1, p // 2]
    got = hecuda.Bfv.innerProductCiphertexts(s.g, lhs, rhs)
    assert np.array_equal(got, o.inner_product(lhs, rhs))


# -------------------------------------------------------------------------------------------------------- decryption
@pytest.mark.parametrize("name", SHAPES)
def test_decrypt_and_noise_budget_at_every_level(shapes, name):
    """Two- and three-polynomial ciphertexts and uniform junk (every branch of the gamma correction) at every level:
    decryption against the oracle, and noiseBudget float-exact against the client oracle."""
    s = shapes(name)
    n, o, sk = s.n, s.o, s.sk.poly
    ms = s.plaintexts(2, 9)
    two = s.encrypt(ms, 80)
    three = o.mul(two[:1], two[1:])
    assert np.array_equal(hecuda.Bfv.decrypt(s.g, two, sk), ms)
    ev = hecuda.Bfv.forwardNtt(s.g, two)
    got = hecuda.Bfv.noiseBudget(s.g, s.sk, ev, evalFormat=True)
    for k in range(2):
        assert got[k] == co.noise_budget(n, s.moduli, s.t, sk, ev[k], eval_format=True) > 0, k
    level = s.L
    while True:
        q = s.q[:level]
        junk2 = orc.fill_uniform(level, q, n, 2 * 2 * level).reshape(2, 2, level, n)
        junk3 = orc.fill_uniform(level + 100, q, n, 3 * level).reshape(1, 3, level, n)
        for cts in (two, three, junk2, junk3):
            got = hecuda.Bfv.decrypt(s.g, cts, sk)
            budgets = hecuda.Bfv.noiseBudget(s.g, s.sk, cts)
            for k in range(len(cts)):
                assert np.array_equal(got[k], o.decrypt(sk, cts[k])), (level, cts.shape, k)
                assert budgets[k] == s.budget(cts[k]), (level, cts.shape, k)
        if level == 1:
            break
        two, three, level = o.mod_switch_down(two), o.mod_switch_down(three), level - 1


# ------------------------------------------------------------------------------------------------------- wire format
@pytest.mark.parametrize("name", SHAPES)
def test_serialize_and_load_at_every_level(shapes, name):
    """serialize / load at skipLSBs 0 and at the largest value every row of the level allows (one bit kept), against
    the reference's packing; one more bit is refused."""
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    polys = orc.fill_uniform(n + 5, q, n, 2 * L).reshape(2, L, n)
    for i, p in enumerate(q):
        polys[0, i, ::3] = p - 1  # the widest field value of every row
    for rows in range(L, 0, -1):
        x = np.ascontiguousarray(polys[:, :rows])
        widest = min(p.bit_length() for p in q[:rows]) - 1
        for skip in (0, widest):
            got = hecuda.Bfv.serialize(s.g, x, skip)
            assert got.shape == (2, opir.serialization_byte_count(n, q[:rows], skip)), (rows, skip)
            assert got[0].tobytes() == opir.serialize_poly(n, q[:rows], x[0], skip), (rows, skip)
            back = hecuda.Bfv.load(s.g, got, rows, skip)
            assert np.array_equal(back, (x >> np.uint64(skip)) << np.uint64(skip)), (rows, skip)
            assert np.array_equal(back[1], opir.load_poly(n, q[:rows], got[1].tobytes(), skip)), (rows, skip)
        with pytest.raises(hecuda.HeError):
            hecuda.Bfv.serialize(s.g, x, widest + 1)


# ------------------------------------------------------------------------------------------------------ Bfv<UInt32>
@pytest.mark.parametrize("name", U32_SETS, ids=[f"{name}-u32" for name in U32_SETS])
def test_word32_operations(shapes, name):
    """Bfv<UInt32> at the sets that support it, against the 32-bit oracle (m~ = 2^16, 29-bit Bsk): the NTT, the multiply
    chain and the fused calls on device encryptions, applyGalois at every level with the generated keys, and the ct x ct
    inner product at 1 and 17 pairs.  Relinearized products and Galois images are decrypted as in the 64-bit tests."""
    s = shapes(name)
    n, q, L, t = s.n, s.q, s.L, s.t
    assert all(p < 1 << 30 for p in s.moduli)
    g, o = hecuda.Context(n, s.moduli, t, scalar=np.uint32), orc.Context(n, s.moduli, t, word_bits=32)
    assert g.auxModuli == g.bskModuli == bb.aux_base(n, s.moduli, t, word_bits=32)[0]
    u32, u64 = (lambda x: x.astype(np.uint32)), (lambda x: x.astype(np.uint64))
    key = hecuda.EvaluationKey32(g, u32(s.relin))
    for el in s.elements:
        key.setGaloisKey(el, u32(s.galois[el]))

    x = orc.fill_uniform(3, q, n, 4 * L).reshape(4, L, n)
    x[0, :, :3] = [[0, 1, p - 1] for p in q]
    fwd = hecuda.Bfv32.forwardNtt(g, u32(x))
    assert np.array_equal(u64(fwd).reshape(-1, n), orc.ntt_forward(n, q, x))
    assert np.array_equal(u64(hecuda.Bfv32.inverseNtt(g, fwd)), x)

    m, sp = s.plaintexts(1, 3)[0], s.sparse(4)
    cts = s.encrypt(np.stack([m, sp]), 90)
    a, b = cts[:1], cts[1:]
    want = negacyclic_times_sparse(m, sp, t)
    product = hecuda.Bfv32.mulAssign(g, u32(a), u32(b))
    assert np.array_equal(u64(product), o.mul(a, b))
    relin = hecuda.Bfv32.relinearize(g, product, key)
    assert np.array_equal(u64(relin), o.relinearize(u64(product), s.relin))
    assert decrypts_to(s, u64(relin)[0], want)
    assert np.array_equal(hecuda.Bfv32.mulRelinearize(g, u32(a), u32(b), key), relin)
    ct, level = relin, L
    while level > 1:
        down = hecuda.Bfv32.modSwitchDown(g, ct)
        assert np.array_equal(u64(down), o.mod_switch_down(u64(ct))), level
        if level == L:
            assert np.array_equal(hecuda.Bfv32.mulRelinearize(g, u32(a), u32(b), key, modSwitchDown=True), down)
            assert np.array_equal(hecuda.Bfv32.relinearizeModSwitchDown(g, product, key), down)
        assert decrypts_to(s, u64(down)[0], want), level
        ct, level = down, level - 1

    ct = np.concatenate([s.encrypt(m[None], 95), orc.fill_uniform(96, q, n, 2 * L).reshape(1, 2, L, n)])
    level = L
    while True:
        for el in s.elements:
            got = u64(hecuda.Bfv32.applyGalois(g, u32(ct), el, key))
            assert np.array_equal(got, o.apply_galois(ct, el, s.galois[el])), (el, level)
            assert decrypts_to(s, got[0], orc.galois_coeff(n, [t], el, m[None])[0]), (el, level)
        if level == 1:
            break
        ct, level = o.mod_switch_down(ct), level - 1

    for terms in IP_TERMS:
        lhs = orc.fill_uniform(terms + 20, q, n, terms * 2 * L).reshape(1, terms, 2, L, n)
        rhs = orc.fill_uniform(terms + 30, q, n, terms * 2 * L).reshape(1, terms, 2, L, n)
        got = hecuda.Bfv32.innerProductCiphertexts(g, u32(lhs), u32(rhs))
        assert np.array_equal(u64(got), o.inner_product(lhs, rhs)), terms
    key.close()
    g.close()


@pytest.mark.parametrize("name", U32_SETS, ids=[f"{name}-u32" for name in U32_SETS])
def test_multiply_at_aligned_operands_u32(name):
    """Bfv<UInt32>'s worst-case multiply over the reference's 29-bit Bsk.  Its floor is exact for the aligned operands
    only while B(L) m_sk > 16 t N q (the second condition of tests/behz_bounds.py); where that fails (t = 40961 and
    65537 over 27 + 28 bits of q) the reference's own floor is not exact for these operands, and the device is checked
    against the oracle only."""
    n, moduli, t = shape_params(name)
    g, o = hecuda.Context(n, moduli, t, scalar=np.uint32), orc.Context(n, moduli, t, word_bits=32)
    q, L, bsk = g.ciphertextModuli, g.L, g.bskModuli
    if math.prod(bsk[:L]) * bsk[L] > 16 * t * n * math.prod(q):
        check_multiply(g, o, n, q, t, word_bits=32)
    else:
        assert t in (40961, 65537)
        a, b = bb.aligned_operands(n, q, 1, 1)[:2]
        got = hecuda.Bfv32.mulAssign(g, a.astype(np.uint32), b.astype(np.uint32)).astype(np.uint64)
        assert np.array_equal(got, o.mul(a, b))
    g.close()
