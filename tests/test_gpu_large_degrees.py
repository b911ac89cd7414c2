"""The BFV operations at N = 2^14 and 2^15, bit-exact against the oracles.

The library runs different code at these degrees than at N <= 8192: the N = 2^15 NTT is split (one cross-half stage,
then two 2^14 transforms), an N = 2^14 row fills a CTA on its own, Galois maps work modulo 2N = 2^15 and 2^16, and the
multiply's auxiliary base, whose conditions take log2 N off both slacks, changes with N.  A host decision or kernel that
is exact for every N <= 8192 and wrong above (a Galois inverse taken modulo 2^14, a bit reversal over 13 bits) passes
every test written at the smaller degrees.  The shapes:

  D14        N = 2^14, bench C3's moduli (8, 55 bits), t = 786433 (SIMD-capable: 2N divides t - 1)
  D15        N = 2^15, 12 moduli of 55 bits (about the 660-bit quantum-128 bound at this degree), t = 786433
  D15-mixed  N = 2^15, rows of 62, 30, 55, h 2^32 + 1, 31 and 61 bits, a 56-bit key-switching modulus: every NTT class,
             and the 62-bit row first, so key switching reduces it into every narrower row (the split NTT's digit path)
  D15-u32    Bfv<UInt32> at N = 2^15 (and 2^14) over 28-29-bit moduli

Each shape asserts the property it was chosen for.  Secret keys, encryptions and evaluation keys are generated on the
device from fixed seeds and compared with the client oracle (at N = 2^15 only the first and last ciphertext of every
key: the oracle's Python sampling of the four whole keys takes about 40 seconds), and every later test uses those keys.
The file runs in about 140 s on one H100."""
import math
import random

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

import behz_bounds as bb  # noqa: E402
import bench  # noqa: E402
import hecuda  # noqa: E402
import threshold_inputs as ti  # noqa: E402
from hecuda import pir  # noqa: E402
from oracle import client_oracle as co  # noqa: E402
from oracle import drbg_oracle as drbg  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from oracle import pir_oracle as opir  # noqa: E402
from rlwe_shapes import (MID, NARROW, NARROW_H, SMALL, WIDE, keyed_elements, mixed_moduli, modulus_class,  # noqa: E402
                         read_device, seed)
from test_gpu_batched_entry_points import chunk_env, stages  # noqa: E402
from test_gpu_behz_bounds import both_signs, check_floor, check_multiply  # noqa: E402
from test_lazy_bounds_model import max_lazy_product_count  # noqa: E402

N14, N15 = 1 << 14, 1 << 15
T = 786433  # 3 * 2^18 + 1, prime
SHAPES = ["D14", "D15", "D15-mixed"]
CHUNK = 3  # HECUDA_CHUNK of the chunked contexts
GiB = 1 << 30


def shape_moduli(name):
    """(N, coefficient moduli) of a 64-bit shape."""
    if name == "D14":
        return N14, list(bench.WORKLOADS["C3"][2])
    if name == "D15":
        return N15, orc.generate_primes([55] * 12, False, N15)
    assert name == "D15-mixed"
    return N15, mixed_moduli(N15)


class Shape:
    """One 64-bit shape: device and oracle contexts, a secret key and an evaluation key (relinearization and
    keyed_elements) generated on the device from fixed seeds, and host copies of the evaluation key."""

    def __init__(self, name):
        self.name = name
        self.n, self.moduli = shape_moduli(name)
        n = self.n
        assert all(p % (2 * n) == 1 for p in self.moduli), "NTT-friendly at this N"
        self.t = T
        assert (T - 1) % (2 * n) == 0
        self.g, self.o = hecuda.Context(n, self.moduli, T), orc.Context(n, self.moduli, T)
        self.L, self.q = self.g.L, self.g.ciphertextModuli
        assert self.g.supportsSimdEncoding
        if name.startswith("D15"):
            assert n == 1 << 15  # the split NTT (fast::kSplitLogN)
        if name == "D15-mixed":
            assert {SMALL, NARROW, NARROW_H, MID, WIDE} <= {modulus_class(p) for p in self.q}
            assert modulus_class(self.q[0]) == WIDE and all(modulus_class(p) != WIDE for p in self.moduli[1:])
        self.elements = keyed_elements(n)
        self.sk = hecuda.SecretKey.generate(self.g, seed(1))
        count = (1 + len(self.elements)) * self.L
        self.a_seeds = [seed(1000 + i) for i in range(count)]
        self.e_seeds = [seed(2000 + i) for i in range(count)]
        self.evk, self.wire = hecuda.EvaluationKey.generate(
            self.g, pir.EvaluationKeyConfig(self.elements, True), self.sk, wire=True, aSeeds=b"".join(self.a_seeds),
            errorSeeds=b"".join(self.e_seeds))
        key_shape = (self.L, 2, self.L + 1, n)
        self.relin = read_device(*self.evk.deviceBuffer()).reshape(key_shape)
        self.galois = {e: read_device(*self.evk.galoisDeviceBuffer(e)).reshape(key_shape) for e in self.elements}
        self._chunked = None

    def chunked(self):
        """(context, key): the same context made with HECUDA_CHUNK=3, and the same evaluation key on it."""
        if self._chunked is None:
            with chunk_env(CHUNK):
                g = hecuda.Context(self.n, self.moduli, self.t)
            key = hecuda.EvaluationKey(g, self.relin)
            for e in self.elements:
                key.setGaloisKey(e, self.galois[e])
            self._chunked = (g, key)
        return self._chunked

    def plaintexts(self, count, rs):
        pts = np.random.default_rng(rs).integers(0, self.t, size=(count, self.n), dtype=np.uint64)
        pts[0, :2] = [0, self.t - 1]
        return pts

    def close(self):
        if self._chunked:
            self._chunked[1].close()
            self._chunked[0].close()
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


# ------------------------------------------------------------------------------------------------------------ client
def key_rows(s):
    """The key ciphertexts compared with the client oracle: all of them at N = 2^14, the first and last at 2^15."""
    return list(range(s.L)) if s.n < N15 else [0, s.L - 1]


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
    assert bytes(poly0[0]) == opir.serialize_poly(n, q, full[0, 0])
    assert np.array_equal(hecuda.Bfv.expandSeeded(s.g, poly0, seeds), full)


@pytest.mark.parametrize("name", SHAPES)
def test_evaluation_key_matches_client_oracle(shapes, name):
    s = shapes(name)
    rows = key_rows(s)
    relin, galois = co.generate_evaluation_key(s.n, s.q, s.moduli[s.L], s.sk.poly, True, s.elements, s.a_seeds,
                                               s.e_seeds, rows)
    assert np.array_equal(s.relin[rows], relin)
    for el in s.elements:
        assert np.array_equal(s.galois[el][rows], galois[el]), el
    loaded = hecuda.EvaluationKey.fromSerialized(s.g, **s.wire)
    assert np.array_equal(read_device(*loaded.deviceBuffer()), s.relin.reshape(-1))
    for el in s.elements:
        assert np.array_equal(read_device(*loaded.galoisDeviceBuffer(el)), s.galois[el].reshape(-1)), el
    loaded.close()


def budgets_match(s, cts):
    got = hecuda.Bfv.noiseBudget(s.g, s.sk, cts)
    for i, ct in enumerate(cts):
        assert got[i] == co.noise_budget(s.n, s.moduli, s.t, s.sk.poly, ct), (ct.shape, i)
    return got


@pytest.mark.parametrize("name", SHAPES)
def test_noise_budget_matches_client_oracle_at_every_level(shapes, name):
    s = shapes(name)
    cts = hecuda.Bfv.encrypt(s.g, s.sk, s.plaintexts(2, 8))
    fresh = budgets_match(s, cts)
    assert np.all(fresh > 0)
    product = hecuda.Bfv.mulAssign(s.g, cts[:1], cts[1:])
    assert budgets_match(s, product)[0] < fresh.min()
    ct, levels = hecuda.Bfv.relinearize(s.g, product, s.evk), 0
    while True:
        budgets_match(s, ct)
        levels += 1
        if ct.shape[-2] == 1:
            break
        ct = hecuda.Bfv.modSwitchDown(s.g, ct)
    assert levels == s.L


# -------------------------------------------------------------------------------------------------------- decryption
@pytest.mark.parametrize("name", SHAPES)
def test_decrypt_at_every_level(shapes, name):
    """Two- and three-polynomial ciphertexts and uniform junk (every branch of the gamma correction) at every level."""
    s = shapes(name)
    n, o, sk = s.n, s.o, s.sk.poly
    ms = s.plaintexts(2, 9)
    fresh = np.stack([o.encrypt(30 + i, sk, m) for i, m in enumerate(ms)])
    assert np.array_equal(hecuda.Bfv.decrypt(s.g, fresh, s.sk), ms)
    three = o.mul(fresh[:1], fresh[1:])
    two = o.relinearize(three, s.relin)
    level = s.L
    while True:
        q = s.q[:level]
        junk2 = orc.fill_uniform(level, q, n, 2 * 2 * level).reshape(2, 2, level, n)
        junk3 = orc.fill_uniform(level + 100, q, n, 3 * level).reshape(1, 3, level, n)
        for cts in (two, three, junk2, junk3):
            got = hecuda.Bfv.decrypt(s.g, cts, sk)
            for k in range(len(cts)):
                assert np.array_equal(got[k], o.decrypt(sk, cts[k])), (level, cts.shape, k)
        if level == s.L:
            assert np.array_equal(hecuda.Bfv.decrypt(s.g, two, sk), hecuda.Bfv.decrypt(s.g, three, sk))
        if level == 1:
            break
        two, three, level = o.mod_switch_down(two), o.mod_switch_down(three), level - 1


def test_decrypt_at_gamma_thresholds_n32768(shapes):
    """tests/threshold_inputs.py's decrypt inputs at N = 2^15.  They solve y_0 modulo gamma (about 2^62) and keep it
    when it is below q_0: about one draw per column when q_0 has 62 bits, 2^7 at 55 bits.  So they are built on
    D15-mixed, whose first row has 62 bits, at the top level and at two moduli."""
    s = shapes("D15-mixed")
    assert s.q[0].bit_length() == 62
    for level in (s.L, 2):
        cts = ti.decrypt_ciphertexts(s.q[:level], s.t, 64, s.n, 2, random.Random(level))
        got = hecuda.Bfv.decrypt(s.g, cts, s.sk)
        for k, ct in enumerate(cts):
            assert np.array_equal(got[k], s.o.decrypt(s.sk.poly, ct)), (level, k)


# ------------------------------------------------------------------------------------------------------------ Galois
@pytest.mark.parametrize("name", SHAPES)
def test_poly_apply_galois_in_both_formats(shapes, name):
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    x = orc.fill_uniform(n + 3, q, n, 2 * L).reshape(2, L, n)
    x[0, :, 0] = 0  # negating zero must stay zero
    for i, p in enumerate(q):
        x[1, i, :4] = [0, 1, p - 1, p // 2]
    ev = hecuda.Bfv.forwardNtt(s.g, x)
    for el in [3, 2 * n - 1] + s.elements:
        got = hecuda.Bfv.polyApplyGalois(s.g, x, el)
        got_ev = hecuda.Bfv.polyApplyGalois(s.g, ev, el, evalFormat=True)
        for k in range(2):
            assert np.array_equal(got[k], orc.galois_coeff(n, q, el, x[k])), (el, k)
            assert np.array_equal(got_ev[k], orc.galois_eval(n, L, el, ev[k])), (el, k)
        assert np.array_equal(hecuda.Bfv.forwardNtt(s.g, got), got_ev), el  # commutes with the NTT


@pytest.mark.parametrize("name", SHAPES)
def test_apply_galois_with_generated_keys(shapes, name):
    """Bfv.applyGalois with the device-generated keys, at the top level and one level down: the oracle's words, and the
    encrypted message permuted."""
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    m = s.plaintexts(1, 10)[0]
    cts = np.stack([s.o.encrypt(40, s.sk.poly, m), orc.fill_uniform(41, q, n, 2 * L).reshape(2, L, n)])
    for el in s.elements:
        want = orc.galois_coeff(n, [s.t], el, m[None])[0]
        for ct in (cts, s.o.mod_switch_down(cts)):
            got = hecuda.Bfv.applyGalois(s.g, ct, el, s.evk)
            assert np.array_equal(got, s.o.apply_galois(ct, el, s.galois[el])), (el, ct.shape)
            assert np.array_equal(hecuda.Bfv.decrypt(s.g, got[:1], s.sk)[0], want), (el, ct.shape)


@pytest.mark.parametrize("name", SHAPES)
def test_multiply_power_of_x(shapes, name):
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    x = orc.fill_uniform(n + 1, q, n, 2 * L).reshape(2, L, n)
    x[0, :, 0] = 0
    for power in (0, 1, -1, n // 2, n, n + 3, -(n + 3), 2 * n, 5 * n + 1, -7 * n - 2):
        got = hecuda.Bfv.multiplyPowerOfX(s.g, x, power)
        for k in range(2):
            assert np.array_equal(got[k], orc.multiply_power_of_x(n, q, power, x[k])), (power, k)


# ------------------------------------------------------------------------------------------------------- wire format
@pytest.mark.parametrize("name", SHAPES)
def test_serialize_load_and_random_polys(shapes, name):
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    polys = orc.fill_uniform(n + 5, q, n, 2 * L).reshape(2, L, n)
    for i, p in enumerate(q):
        polys[0, i, ::3] = p - 1  # the widest field value of every row
    for rows in (L, 1):
        for skip in sorted({0, 1, 5, min(p.bit_length() for p in q[:rows]) - 2}):
            x = np.ascontiguousarray(polys[:, :rows])
            got = hecuda.Bfv.serialize(s.g, x, skip)
            assert got.shape == (2, opir.serialization_byte_count(n, q[:rows], skip))
            assert got[0].tobytes() == opir.serialize_poly(n, q[:rows], x[0], skip), (rows, skip)
            back = hecuda.Bfv.load(s.g, got, rows, skip)
            assert np.array_equal(back, (x >> np.uint64(skip)) << np.uint64(skip)), (rows, skip)
            assert np.array_equal(back[1], opir.load_poly(n, q[:rows], got[1].tobytes(), skip)), (rows, skip)
    seeds = np.random.default_rng(n).integers(0, 256, size=(2, 32), dtype=np.uint8)
    assert 16 * n > drbg.BUFFER_COUNT  # every row spans many 4096-byte DRBG generates
    for rows in (L, 1):
        got = hecuda.Bfv.randomPolys(s.g, seeds, rows)
        for b in range(2):
            assert np.array_equal(got[b], drbg.random_poly(n, q[:rows], seeds[b].tobytes())), (rows, b)


# ---------------------------------------------------------------------------------------------------- inner products
@pytest.mark.parametrize("name", SHAPES)
def test_ct_pt_inner_product(shapes, name):
    """33 terms, with and without a `present` mask, all-(q_i - 1) and uniform operands.  With a 62-bit row (D15-mixed)
    the lazy accumulator holds 16 products of (q - 1)^2, so 33 terms pass its reduction interval twice; with 55-bit rows
    the interval is 2^18 terms and the test is plain parity."""
    s = shapes(name)
    n, q, L = s.n, s.q, s.L
    terms, rows = 33, 2
    cap = max_lazy_product_count(max(q))
    assert (2 * cap < terms) == (max(q).bit_length() == 62)
    if 2 * cap < terms:
        assert (cap + 1) * (max(q) - 1) ** 2 >= 1 << 128
    top_c = np.stack([np.full((terms, 2, n), p - 1, dtype=np.uint64) for p in q], axis=2)
    top_p = np.stack([np.full((rows, terms, n), p - 1, dtype=np.uint64) for p in q], axis=2)
    uniform_c = orc.fill_uniform(terms, q, n, terms * 2 * L).reshape(terms, 2, L, n)
    uniform_p = orc.fill_uniform(terms + 1, q, n, rows * terms * L).reshape(rows, terms, L, n)
    present = np.ones((rows, terms), dtype=np.uint8)
    present[0, [15, 16, 17]] = 0  # nil on and next to a reduction
    present[1, ::3] = 0
    for cts, pts in ((top_c, top_p), (uniform_c, uniform_p)):
        for pres in (None, present):
            got = hecuda.Bfv.innerProduct(s.g, cts, pts, pres)
            assert np.array_equal(got, s.o.inner_product_plain(cts, pts, pres)), pres is None


def ip_moduli():
    """The four largest 55-bit primes = 1 mod 2^16: NTT-friendly at N = 2^14 and 2^15."""
    return orc.generate_primes([55] * 4, False, N15)


def t_for_pair_cap(n, moduli, cap):
    """The largest t whose auxiliary pair cap at this N is still at least `cap` (the cap only falls as t grows, until
    the auxiliary base is given up for Bsk)."""
    lo, hi = 2, min(bb.ciphertext_moduli(moduli)) - 1
    assert cap <= bb.aux_pair_cap(n, moduli, lo) < math.inf
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if cap <= bb.aux_pair_cap(n, moduli, mid) < math.inf else (lo, mid)
    return lo


@pytest.mark.parametrize("n", [N14, N15])
def test_ct_ct_inner_product_across_the_pair_bound(n):
    """Bfv.innerProductCiphertexts at 1, cap, cap + 1 and 2 * fast_wrap aligned pairs, with t chosen so that the pair
    cap (bb.aux_pair_cap: past it the sum runs over Bsk) is small at this N.  The last count is only right if the call
    left the auxiliary base.

    The limit of this test: the cap keeps about 5 bits below the sum's real wrap (fast_wrap is about 32 times the cap),
    and the library does not report its cap.  So a device cap that is wrong by less than that factor -- log2 N taken
    as 13 at N = 2^15 makes it 4 times too large -- gives the same results and is not caught here.  Device memory: the
    inputs and (4P + 3)(2L + 1)N words of scratch."""
    moduli = ip_moduli()
    t = t_for_pair_cap(n, moduli, 4)
    cap, wrap = bb.aux_pair_cap(n, moduli, t), bb.fast_wrap(n, moduli, t)
    assert 4 <= cap <= 16 and 2 * wrap > cap + 1
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    q, L = g.ciphertextModuli, g.L
    assert g.auxModuli == bb.aux_base(n, moduli, t)[0] != g.bskModuli
    for P in sorted({1, cap, cap + 1, 2 * wrap}):
        words = 2 * P * 2 * L * n + (4 * P + 3) * (2 * L + 1) * n + 3 * L * n
        assert 8 * words < 8 * GiB, P
        lhs, rhs, _ = bb.aligned_operands(n, q, P, 1)
        got = hecuda.Bfv.innerProductCiphertexts(g, lhs[None], rhs[None])
        assert np.array_equal(got, o.inner_product(lhs[None], rhs[None])), P
        check_floor(got[0], q, t, lhs[0], rhs[0], scale=P)
        del lhs, rhs
    g.close()


# ------------------------------------------------------------------------------------------------------------ multiply
@pytest.mark.parametrize("name", ["D14", "D15"])
@pytest.mark.parametrize("which", ["t", "largest-fast-t", "largest-fast-t+1"])
def test_multiply_at_aligned_operands(name, which):
    """Bfv.mulAssign at operands whose lifts are all +-(q/2 - q/2^16) and whose products' N terms share a sign, at the
    shape's t, at the largest t that keeps the auxiliary base at this N, and at the next t, which leaves it."""
    n, moduli = shape_moduli(name)
    fast_t = bb.largest_fast_t(n, moduli)
    t = {"t": T, "largest-fast-t": fast_t, "largest-fast-t+1": fast_t + 1}[which]
    assert t < min(bb.ciphertext_moduli(moduli))
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    aux, bsk = bb.aux_base(n, moduli, t)
    assert g.auxModuli == aux and g.bskModuli == bsk
    if which == "largest-fast-t+1":
        assert aux != bb.aux_base(n, moduli, fast_t)[0]
    else:
        assert aux != bsk
    check_multiply(g, o, n, g.ciphertextModuli, t)
    g.close()


def u32_moduli(n):
    return orc.generate_primes([28, 28, 29, 29], False, n)


@pytest.mark.parametrize("n", [N14, N15])
@pytest.mark.parametrize("t", [17, T])
def test_multiply_at_aligned_operands_u32(n, t):
    """Bfv<UInt32> multiplies over the reference's Bsk of 29-bit primes.  Its floor is exact for the aligned operands
    only while B(L) m_sk > 16 t N q (the second condition of tests/behz_bounds.py): over 85 bits of q at N >= 2^14 that
    needs t < 2^12.  So the floor is checked at t = 17; at t = 786433 the reference's own floor is not exact for these
    operands, and the device is checked against the oracle only."""
    moduli = u32_moduli(n)
    g, o = hecuda.Context(n, moduli, t, scalar=np.uint32), orc.Context(n, moduli, t, word_bits=32)
    q, L, bsk = g.ciphertextModuli, g.L, g.bskModuli
    assert g.auxModuli == bsk == bb.aux_base(n, moduli, t, word_bits=32)[0]
    exact = math.prod(bsk[:L]) * bsk[L] > 16 * t * n * math.prod(q)
    assert exact == (t == 17)
    if exact:
        check_multiply(g, o, n, q, t, word_bits=32)
    else:
        a, b = both_signs(n, q)
        got = hecuda.Bfv32.mulAssign(g, a.astype(np.uint32), b.astype(np.uint32)).astype(np.uint64)
        assert np.array_equal(got, o.mul(a, b))
    g.close()


# --------------------------------------------------------------------------------------- fused calls across chunks
def launches(fn):
    torch.cuda.synchronize()
    before = hecuda.kernel_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, hecuda.kernel_launch_count() - before


@pytest.mark.parametrize("batch", [1, 7])
@pytest.mark.parametrize("name", SHAPES)
def test_fused_calls_across_chunk_boundaries(shapes, name, batch):
    """mulRelinearize (+ modSwitchDown), relinearizeModSwitchDown, applyGalois and both inner products on a context made
    with HECUDA_CHUNK=3: equal to the oracle and to the same call on the default context.  The calls sized by the chunk
    run in ceil(batch / items per stage) stages, which at batch 7 is at least two, each launching what a one-item call
    launches.  The ct x pt inner product is staged by its own word budget and runs whole here."""
    s = shapes(name)
    g3, key3 = s.chunked()
    n, q, L, o = s.n, s.q, s.L, s.o
    pairs, terms = 2, 3
    a = orc.fill_uniform(batch, q, n, batch * 2 * L).reshape(batch, 2, L, n)
    b = orc.fill_uniform(batch + 10, q, n, batch * 2 * L).reshape(batch, 2, L, n)
    lhs = orc.fill_uniform(batch + 20, q, n, batch * pairs * 2 * L).reshape(batch, pairs, 2, L, n)
    rhs = orc.fill_uniform(batch + 30, q, n, batch * pairs * 2 * L).reshape(batch, pairs, 2, L, n)
    cts = orc.fill_uniform(batch + 40, q, n, terms * 2 * L).reshape(terms, 2, L, n)
    pts = orc.fill_uniform(batch + 50, q, n, batch * terms * L).reshape(batch, terms, L, n)
    product = o.mul(a, b)
    relin = o.relinearize(product, s.relin)
    down = o.mod_switch_down(relin)
    # (label, call on (context, key, items), expected, items per stage of the chunked context or None)
    ops = [
        ("mulRelinearize", lambda g, k, i: hecuda.Bfv.mulRelinearize(g, a[i], b[i], k), relin, max(1, CHUNK // 2)),
        ("mulRelinearize+modSwitchDown",
         lambda g, k, i: hecuda.Bfv.mulRelinearize(g, a[i], b[i], k, modSwitchDown=True), down, max(1, CHUNK // 2)),
        ("relinearizeModSwitchDown", lambda g, k, i: hecuda.Bfv.relinearizeModSwitchDown(g, product[i], k), down,
         CHUNK),
        ("innerProductCiphertexts", lambda g, k, i: hecuda.Bfv.innerProductCiphertexts(g, lhs[i], rhs[i]),
         o.inner_product(lhs, rhs), max(1, CHUNK // pairs)),
        ("innerProduct", lambda g, k, i: hecuda.Bfv.innerProduct(g, cts, pts[i]), o.inner_product_plain(cts, pts),
         None),
    ]
    for el in s.elements:  # rotate-by-1's inverse is 3 at every N; the other two inverses change with N
        ops.append((f"applyGalois {el}", lambda g, k, i, el=el: hecuda.Bfv.applyGalois(g, a[i], el, k),
                    o.apply_galois(a, el, s.galois[el]), CHUNK))
    everything, first = slice(None), slice(0, 1)
    for label, call, want, per_stage in ops:
        got3, count = launches(lambda: call(g3, key3, everything))
        assert np.array_equal(got3, want), f"{label}, HECUDA_CHUNK={CHUNK}"
        assert np.array_equal(call(s.g, s.evk, everything), want), f"{label}, default chunk"
        if per_stage is not None:
            staged = stages(batch, per_stage)
            assert staged >= (2 if batch == 7 else 1), label
            _, base = launches(lambda: call(g3, key3, first))
            assert count == staged * base, (label, count, staged, base)


# ------------------------------------------------------------------------------------------------------ Bfv<UInt32>
@pytest.mark.parametrize("n", [N14, N15])
def test_word32_operations(n):
    """Bfv<UInt32>: the NTT, multiply, relinearize, modSwitchDown, applyGalois and the ct x ct inner product against the
    32-bit oracle (m~ = 2^16, gamma = 2^30 - 20405, 29-bit Bsk)."""
    moduli = u32_moduli(n)
    g, o = hecuda.Context(n, moduli, T, scalar=np.uint32), orc.Context(n, moduli, T, word_bits=32)
    L, q = g.L, g.ciphertextModuli
    assert all(p < 1 << 30 and p % (2 * n) == 1 for p in moduli)
    x = orc.fill_uniform(3, q, n, 4 * L).reshape(4, L, n)
    x[0, :, :3] = [[0, 1, p - 1] for p in q]
    fwd = hecuda.Bfv32.forwardNtt(g, x.astype(np.uint32))
    assert np.array_equal(fwd.astype(np.uint64).reshape(-1, n), orc.ntt_forward(n, q, x))
    assert np.array_equal(hecuda.Bfv32.inverseNtt(g, fwd).astype(np.uint64), x)
    batch = 3
    a = orc.fill_uniform(11, q, n, batch * 2 * L).reshape(batch, 2, L, n)
    b = orc.fill_uniform(12, q, n, batch * 2 * L).reshape(batch, 2, L, n)
    for i, p in enumerate(q):
        a[0, :, i, :4] = p - 1
        b[0, :, i, :4] = [0, 1, p - 1, p // 2]
    a32, b32 = a.astype(np.uint32), b.astype(np.uint32)
    prod = hecuda.Bfv32.mulAssign(g, a32, b32)
    want = o.mul(a, b)
    assert np.array_equal(prod.astype(np.uint64), want)
    sk, rk = o.keygen(5)
    key = hecuda.EvaluationKey32(g, rk.astype(np.uint32))
    relin = hecuda.Bfv32.relinearize(g, prod, key)
    want_relin = o.relinearize(want, rk)
    assert np.array_equal(relin.astype(np.uint64), want_relin)
    assert np.array_equal(hecuda.Bfv32.modSwitchDown(g, relin).astype(np.uint64), o.mod_switch_down(want_relin))
    m = np.random.default_rng(n).integers(0, T, size=n, dtype=np.uint64)
    cts = np.stack([o.encrypt(6, sk, m), a[1]])
    for el in keyed_elements(n):
        gk = o.galois_keygen(77 + el % 1000, sk, el)
        key.setGaloisKey(el, gk.astype(np.uint32))
        got = hecuda.Bfv32.applyGalois(g, cts.astype(np.uint32), el, key).astype(np.uint64)
        assert np.array_equal(got, o.apply_galois(cts, el, gk)), el
        assert np.array_equal(o.decrypt(sk, got[0]), orc.galois_coeff(n, [T], el, m[None])[0]), el
    lhs, rhs = a[:2].reshape(1, 2, 2, L, n), b[:2].reshape(1, 2, 2, L, n)
    got = hecuda.Bfv32.innerProductCiphertexts(g, lhs.astype(np.uint32), rhs.astype(np.uint32)).astype(np.uint64)
    assert np.array_equal(got, o.inner_product(lhs, rhs))
    key.close()
    g.close()
