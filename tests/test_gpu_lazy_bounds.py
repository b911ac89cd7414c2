"""The lazy accumulators on the GPU at their bounds: key switching whose sums pass (2^64 - p) 2^64 (62-bit moduli,
l >= 13), ct x pt scans past maxLazyProductAccumulationCount terms, ct x ct sums past their pair cap, the MulPir scans
over uint32 and uint64 database rows, and NTT launches whose row lists mix every modulus class.

Every case computes, with exact Python integers, the largest sum its operands put into an accumulator and asserts that
it crosses the bound the case is about: a case that silently stays below its bound tests nothing."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir
from oracle import oracle as orc
from oracle import pir_oracle as opir
from rlwe_shapes import MID, NARROW, NARROW_H, SMALL, WIDE, mixed_moduli, modulus_class
from test_lazy_bounds_model import (U128, constant_target, first_window_sum, ip_plain_model, ks_mac_reduces_high_word,
                                    ks_mac_wraps_without_high_reduction, ks_model, max_lazy_product_count,
                                    saturated_key, tensor_sum_cap)

TEST_MODULI_BITS = [55, 52, 62, 58]  # TestUtils.testCoefficientModuli for UInt64 (TestUtilities.swift:312-317)
TILE = 4  # clients per thread of the first-dimension scan (kScanClientTile)


def primes(bits, count, n):
    return orc.generate_primes([bits] * count, False, n)


# ------------------------------------------------------------------------------------------------ key switching
def ks_widest(o, target_rows, key):
    """The largest digit x key sum of one key switch of `target_rows` (l, N), with its row's modulus."""
    return ks_model(o, target_rows, key)[1]


def product_for_constant_c2(o, value):
    """Top-level ciphertexts a, b (Coeff) whose product's third polynomial is about `value` in coefficient 0 and zero
    elsewhere: a1 = b1 = the constant A with t A^2 / Q close to `value`."""
    import math

    n, L = o.n, o.L
    Q = math.prod(o.q)
    A = math.isqrt(value * Q // o.t)
    a = orc.fill_uniform(71, o.q, n, 2 * L).reshape(1, 2, L, n)
    b = orc.fill_uniform(72, o.q, n, 2 * L).reshape(1, 2, L, n)
    for i, q in enumerate(o.q):
        a[0, 1, i, :], b[0, 1, i, :] = 0, 0
        a[0, 1, i, 0], b[0, 1, i, 0] = A % q, A % q
    return a, b


@pytest.mark.parametrize("n", [16, 4096])
@pytest.mark.parametrize("L", [14, 13, 12])
def test_keyswitch_at_the_accumulator_bound(n, L):
    """62-bit moduli; every key residue m_r - 1 and target rows min m_r - 1 in coefficient 0, so every digit is about
    m_r - 1.  At l >= 13 the sums pass (2^64 - p) 2^64, where one Montgomery reduction alone would return a value
    above 2^64; l = 12 is the control."""
    moduli = primes(62, L + 1, n)
    t = orc.generate_primes([17], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    key_rows = saturated_key(moduli, L, n)
    key = hecuda.EvaluationKey(g, key_rows)
    element = 3
    key.setGaloisKey(element, key_rows)
    top = min(moduli) - 1
    batch = 2
    for l in sorted({L, 13, 12} & set(range(1, L + 1)), reverse=True):
        q = moduli[:l]
        target = constant_target(moduli, l, n, top)
        widest = ks_widest(o, target, key_rows)
        assert ks_mac_wraps_without_high_reduction(widest) == (l >= 13) and ks_mac_reduces_high_word(widest), f"l={l}"
        ct3 = orc.fill_uniform(l, q, n, batch * 3 * l).reshape(batch, 3, l, n)
        ct3[:, 2] = target
        want = o.relinearize(ct3, key_rows)
        assert np.array_equal(hecuda.Bfv.relinearize(g, ct3, key), want), f"relinearize l={l}"
        down = o.mod_switch_down(want)
        assert np.array_equal(hecuda.Bfv.relinearizeModSwitchDown(g, ct3, key), down), f"relinearizeModSwitchDown l={l}"
        assert np.array_equal(hecuda.Bfv.modSwitchDown(g, want), down)
        ct2 = np.ascontiguousarray(ct3[:, :2])
        ct2[:, 1] = target  # x -> x^3 keeps a constant polynomial: the switched target is the same
        got = hecuda.Bfv.applyGalois(g, ct2, element, key)
        assert np.array_equal(got, o.apply_galois(ct2, element, key_rows)), f"applyGalois l={l}"
    # the fused multiply: its third polynomial is the constant about min m_r - 3
    a, b = product_for_constant_c2(o, top - 2)
    prod = o.mul(a, b)
    assert not prod[0, 2, :, 1:].any()
    assert ks_mac_wraps_without_high_reduction(ks_widest(o, prod[0, 2], key_rows)) == (L >= 13)
    relin = o.relinearize(prod, key_rows)
    assert np.array_equal(hecuda.Bfv.mulRelinearize(g, a, b, key), relin)
    assert np.array_equal(hecuda.Bfv.mulRelinearize(g, a, b, key, modSwitchDown=True), o.mod_switch_down(relin))
    key.close()
    g.close()


def test_keyswitch_with_a_real_key_at_fifteen_62_bit_moduli():
    """The reference's largest context at 62 bits (15 moduli) end to end: Dec(mulRelinearize(Enc(m1), Enc(m2))) = m1 m2,
    relinearized and switched down, and bit-identical to the oracle."""
    n = 4096
    moduli = primes(62, 15, n)
    assert len(moduli) == max_lazy_product_count(max(moduli)) - 1
    t = orc.generate_primes([20], True, n)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    sk, rk = o.keygen(41)
    key = hecuda.EvaluationKey(g, rk)
    rnd = random.Random(15)
    m1 = np.array([rnd.randrange(t) for _ in range(n)], dtype=np.uint64)
    m2 = np.zeros(n, dtype=np.uint64)
    m2[0], m2[7], m2[n - 1] = 2, t - 1, 9
    c1, c2 = o.encrypt(1, sk, m1)[None], o.encrypt(2, sk, m2)[None]
    relin = o.relinearize(o.mul(c1, c2), rk)
    assert np.array_equal(hecuda.Bfv.mulRelinearize(g, c1, c2, key), relin)
    down = hecuda.Bfv.mulRelinearize(g, c1, c2, key, modSwitchDown=True)
    assert np.array_equal(down, o.mod_switch_down(relin))
    expect = [0] * n
    m1l = [int(v) for v in m1]
    for j, c in ((0, 2), (7, t - 1), (n - 1, 9)):
        for i in range(n):
            k = i + j
            if k < n:
                expect[k] = (expect[k] + m1l[i] * c) % t
            else:
                expect[k - n] = (expect[k - n] - m1l[i] * c) % t
    assert o.decrypt(sk, relin[0]).tolist() == expect
    assert o.decrypt(sk, down[0]).tolist() == expect
    key.close()
    g.close()


@pytest.mark.parametrize("n", [16, 4096])
def test_keyswitch_saturated_operands_u32(n):
    """The same saturated key and target rows through Bfv<UInt32> at 15 moduli of 30 bits (its largest context)."""
    moduli = primes(30, 15, n)
    assert len(moduli) == max_lazy_product_count(max(moduli), 64) - 1
    t = 17
    g, o = hecuda.Context(n, moduli, t, scalar=np.uint32), orc.Context(n, moduli, t, word_bits=32)
    L = len(moduli) - 1
    key_rows = saturated_key(moduli, L, n)
    key = hecuda.EvaluationKey32(g, key_rows)
    element = 3
    key.setGaloisKey(element, key_rows)
    top = min(moduli) - 1
    for l in (L, L - 1):
        ct3 = orc.fill_uniform(l, moduli[:l], n, 2 * 3 * l).reshape(2, 3, l, n)
        ct3[:, 2] = constant_target(moduli, l, n, top)
        want = o.relinearize(ct3, key_rows)
        assert np.array_equal(hecuda.Bfv32.relinearize(g, ct3, key).astype(np.uint64), want)
        assert np.array_equal(hecuda.Bfv32.relinearizeModSwitchDown(g, ct3, key).astype(np.uint64), o.mod_switch_down(want))
        ct2 = np.ascontiguousarray(ct3[:, :2])
        ct2[:, 1] = ct3[:, 2]
        assert np.array_equal(hecuda.Bfv32.applyGalois(g, ct2, element, key).astype(np.uint64),
                              o.apply_galois(ct2, element, key_rows))
    key.close()
    g.close()


def test_context_moduli_count_limit():
    """Context.swift:114-124: a key-switching context needs fewer moduli than maxLazyProductAccumulationCount."""
    n = 16
    for bits, scalar, double_bits in ((62, np.uint64, 128), (30, np.uint32, 64)):
        moduli = primes(bits, 16, n)
        assert max_lazy_product_count(max(moduli), double_bits) == 16
        hecuda.Context(n, moduli[:15], 17, scalar=scalar).close()
        with pytest.raises(hecuda.HeError) as err:
            hecuda.Context(n, moduli, 17, scalar=scalar)
        assert "invalidEncryptionParameters" in str(err.value)
    # no key-switching context, no limit on the count: one modulus
    hecuda.Context(n, primes(62, 1, n), 17).close()


# ------------------------------------------------------------------------------------------------ ct x pt scan
@pytest.mark.parametrize("n", [16, 4096])
@pytest.mark.parametrize("terms", [15, 16, 17, 32, 33, 48])
def test_ct_pt_inner_product_past_max_terms(n, terms):
    moduli = primes(62, 4, n)
    g, o = hecuda.Context(n, moduli, 65537), orc.Context(n, moduli, 65537)
    L, rows = o.L, 3
    q = moduli[:L]
    cap = max_lazy_product_count(max(q))
    assert cap == 16
    uniform_c = orc.fill_uniform(terms, q, n, terms * 3 * L).reshape(terms, 3, L, n)
    uniform_p = orc.fill_uniform(terms + 100, q, n, rows * terms * L).reshape(rows, terms, L, n)
    top_c = np.stack([np.full((terms, 3, n), m - 1, dtype=np.uint64) for m in q], axis=2)
    top_p = np.stack([np.full((rows, terms, n), m - 1, dtype=np.uint64) for m in q], axis=2)
    present = np.ones((rows, terms), dtype=np.uint8)
    present[1, [k for k in (cap - 1, cap, cap + 1, 2 * cap - 1, 2 * cap) if k < terms]] = 0  # nil on / next to a reduction
    present[2, ::3] = 0
    for cts, pts, extreme in ((top_c, top_p, True), (uniform_c, uniform_p, False)):
        for polys in (1, 2, 3):
            for l in (L, 2):
                c = np.ascontiguousarray(cts[:, :polys, :l])
                p = np.ascontiguousarray(pts[:, :, :l])
                for pres in (None, present):
                    want = o.inner_product_plain(c, p, pres)
                    # the exact model on the first 16 columns (all of them at N = 16)
                    model, prods = ip_plain_model(c[..., :16], p[..., :16], q[:l], pres)
                    assert np.array_equal(want[..., :16], model)
                    if extreme and pres is None:
                        assert (first_window_sum(prods, cap + 1) >= U128) == (terms > cap)
                    got = hecuda.Bfv.innerProduct(g, c, p, pres)
                    assert np.array_equal(got, want), (polys, l, pres is None)
    g.close()


# ------------------------------------------------------------------------------------------------ ct x ct sum
@pytest.mark.parametrize("bits,pairs", [(62, 4), (62, 5), (62, 7), (62, 8), (62, 9), (61, 16), (61, 17), (61, 31)])
@pytest.mark.parametrize("n", [16, 4096])
@pytest.mark.parametrize("aux", ["fast", "reference"])
def test_ct_ct_inner_product_past_max_pairs(bits, pairs, n, aux, monkeypatch):
    moduli = primes(bits, 3, n)
    t = orc.generate_primes([12], True, 1)[0]
    if aux == "reference":
        monkeypatch.setenv("HECUDA_AUX_BASE", "reference")
    g = hecuda.Context(n, moduli, t)
    monkeypatch.delenv("HECUDA_AUX_BASE", raising=False)
    o = orc.Context(n, moduli, t)
    L, groups = o.L, 2
    lhs = orc.fill_uniform(bits + pairs, moduli[:L], n, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, n)
    rhs = orc.fill_uniform(bits - pairs, moduli[:L], n, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, n)
    for i in range(L):  # group 0: q_i - 1 in coefficient 0, so every Eval value of the Q rows is q_i - 1
        lhs[0, :, :, i, :], rhs[0, :, :, i, :] = 0, 0
        lhs[0, :, :, i, 0], rhs[0, :, :, i, 0] = moduli[i] - 1, moduli[i] - 1
    pmax = max(moduli[:L] + (g.bskModuli if aux == "reference" else g.auxModuli))
    assert pmax == max(moduli[:L])
    widest = pairs * 2 * (pmax - 1) ** 2  # the middle sum of a Q row of group 0
    assert (widest >= 1 << 127) == (pairs > tensor_sum_cap(pmax))
    if pairs == 2 * tensor_sum_cap(pmax) - 1:  # under a cap twice as large, one Montgomery reduction would wrap
        assert widest >= ((1 << 64) - pmax) << 64
    assert np.array_equal(hecuda.Bfv.innerProductCiphertexts(g, lhs, rhs), o.inner_product(lhs, rhs))
    g.close()


# ------------------------------------------------------------------------------------------------ MulPir scans
class Setup:
    """One MulPir server (context, parameter, database) and its oracle twin (as in test_gpu_pir_clients.py)."""

    def __init__(self, g, o, entries, entry_size, seed):
        self.g, self.o = g, o
        self.rng = random.Random(seed)
        config = (entries, entry_size, 1, 1, False, "noCompression", False)
        self.param = pir.MulPir.generateParameter(pir.IndexPirConfig(*config), g)
        self.oparam = opir.generate_parameter(opir.IndexPirConfig(*config), o.n, o.t)
        assert self.param.dimensions == self.oparam.dimensions
        self.db = [bytes(self.rng.randrange(256) for _ in range(entry_size)) for _ in range(entries)]
        self.server = pir.MulPirServer(self.param, g, [pir.MulPirServer.process(self.db, g, self.param)])
        self.odb = opir.process_database(o, self.oparam, self.db)
        self.entries = entries

    def client(self, seed):
        o = self.o
        sk, relin = o.keygen(seed)
        key = hecuda.EvaluationKey(self.g, relin)
        okeys = {}
        for i, e in enumerate(self.param.evaluationKeyConfig.galoisElements):
            okeys[e] = o.galois_keygen(7000 + 31 * seed + i, sk, e)
            key.setGaloisKey(e, okeys[e])
        indices = [self.rng.randrange(self.entries)]
        query = np.stack(opir.generate_query(o, self.oparam, indices, sk, 9000 + seed))
        return dict(sk=sk, relin=relin, key=key, okeys=okeys, indices=indices, query=query)

    def widest_scan_sum(self, c):
        """The largest unreduced first-dimension sum sum_k query_k pt_k of client c, over rows, polys and columns."""
        o, dim0 = self.o, self.param.dimensions[0]
        expanded = opir.expand(o, list(c["query"]), self.oparam.expanded_query_count, c["okeys"])
        first = np.stack([np.stack([orc.ntt_forward(o.n, o.q, ct[p]) for p in range(2)]) for ct in expanded[:dim0]])
        pts = self.odb.plaintexts[:dim0].astype(object)
        return max(int(sum(first[k, p].astype(object) * pts[k] for k in range(dim0)).max()) for p in range(2))

    def check(self, clients):
        got = self.server.computeResponses(np.stack([c["query"] for c in clients]), [c["key"] for c in clients])
        for j, c in enumerate(clients):
            expected = opir.compute_response(self.o, list(c["query"]), 1, c["okeys"], c["relin"], [self.odb], self.oparam)
            assert np.array_equal(got[j, 0, 0], expected[0][0]), f"client {j}"
            reply = [[got[j, 0, 0]]]
            assert opir.decrypt_response(self.o, self.oparam, reply, c["indices"], c["sk"]) == [self.db[c["indices"][0]]]
        return got


@pytest.mark.parametrize("bits,entries,entry_size,t,double_bits,cap", [
    ([31, 31, 31], 64, 8, 17, 64, 4),        # uint32 database rows, reduced every 4 terms
    ([30, 30, 30], 128, 8, 17, 64, 16),      # uint32 database rows, every 16
    (TEST_MODULI_BITS, 128, 20, 1153, 128, 16),  # uint64 rows (a 62-bit modulus), every 16
])
@pytest.mark.parametrize("count", [1, TILE + 1])
def test_mulpir_scan_past_max_terms(bits, entries, entry_size, t, double_bits, cap, count):
    n = 16
    moduli = orc.generate_primes(bits, False, n)
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    assert max_lazy_product_count(max(o.q), double_bits) == cap
    s = Setup(g, o, entries, entry_size, seed=entries + count)
    dim0 = s.param.dimensions[0]
    assert s.param.dimensions == [entries] and dim0 >= 4 * cap
    clients = [s.client(50 + c) for c in range(count)]
    for c in clients:  # without its in-loop reductions the scan's accumulator would wrap
        assert s.widest_scan_sum(c) >= 1 << double_bits
    s.check(clients)
    for c in clients:
        c["key"].close()
    g.close()


# ------------------------------------------------------------------------------------------------ NTT classes
def edge_inputs(moduli, n, seed, batch_extra=1):
    """(4 + batch_extra, rows, N): all p - 1, alternating 0 / p - 1, a delta, and uniform rows."""
    rows = len(moduli)
    x = np.zeros((3, rows, n), dtype=np.uint64)
    for r, p in enumerate(moduli):
        x[0, r, :] = p - 1
        x[1, r, 1::2] = p - 1
        x[2, r, 0] = 1
    u = orc.fill_uniform(seed, moduli, n, batch_extra * rows).reshape(batch_extra, rows, n)
    return np.concatenate([x, u])


@pytest.mark.parametrize("n", [1024, 8192, 16384, 32768])
def test_ntt_launches_mixing_every_class(n):
    moduli = mixed_moduli(n)
    t = orc.generate_primes([12], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    L = o.L
    bases = {
        hecuda.BASE_Q: moduli[:L],
        hecuda.BASE_Q_BSK: moduli[:L] + g.bskModuli,
        hecuda.BASE_KEYSWITCH: moduli[:L] + [moduli[L]],
    }
    for base, rows in bases.items():
        assert {SMALL, NARROW, NARROW_H, MID, WIDE} <= {modulus_class(p) for p in rows}, base
        x = edge_inputs(rows, n, base + 7)
        fwd = hecuda.Bfv.forwardNtt(g, x, base)
        assert np.array_equal(fwd.reshape(-1, n), orc.ntt_forward(n, rows, x)), base
        assert np.all(fwd[2] == 1)
        assert np.array_equal(hecuda.Bfv.inverseNtt(g, fwd, base), x), base
        assert np.array_equal(hecuda.Bfv.inverseNtt(g, x, base).reshape(-1, n), orc.ntt_inverse(n, rows, x)), base
    # key switching: the 62-bit target row 0 is reduced into every narrower row's modulus before its NTT
    assert modulus_class(moduli[0]) == WIDE and {modulus_class(p) for p in moduli[1:]} >= {SMALL, NARROW, NARROW_H, MID}
    _, rk = o.keygen(n % 997)
    key = hecuda.EvaluationKey(g, rk)
    ct3 = orc.fill_uniform(n % 991, moduli[:L], n, 2 * 3 * L).reshape(2, 3, L, n)
    for i in range(L):
        ct3[0, 2, i, :] = moduli[i] - 1
    want = o.relinearize(ct3, rk)
    assert np.array_equal(hecuda.Bfv.relinearize(g, ct3, key), want)
    assert np.array_equal(hecuda.Bfv.relinearize(g, ct3[:, :, :3], key), o.relinearize(ct3[:, :, :3], rk))
    key.close()
    g.close()


@pytest.mark.parametrize("n", [2, 4, 8, 16, 32, 64, 256, 1024, 2048, 4096, 8192, 16384, 32768])
def test_ntt_matches_oracle_62_bit(n):
    """test_ntt_matches_oracle (test_gpu_parity.py) for the WIDE class: 62-bit moduli through the device kernels."""
    moduli = primes(62, 3, n)
    assert all(modulus_class(p) == WIDE for p in moduli)
    g = hecuda.Context(n, moduli, 2)
    x = orc.fill_uniform(n + 62, moduli[:2], n, 2 * 5).reshape(5, 2, n)
    fwd = hecuda.Bfv.forwardNtt(g, x, hecuda.BASE_Q)
    assert np.array_equal(fwd.reshape(-1, n), orc.ntt_forward(n, moduli[:2], x))
    assert np.array_equal(hecuda.Bfv.inverseNtt(g, fwd, hecuda.BASE_Q), x)
    for p in moduli[:2]:
        edge = np.zeros((4, n), dtype=np.uint64)
        edge[1, :] = p - 1
        edge[2, 0] = 1
        edge[3, 1::2] = p - 1
        out = hecuda.Bfv.forwardNttRows(g, p, edge)
        assert np.array_equal(out, orc.ntt_forward(n, [p], edge))
        assert np.all(out[2] == 1)
        assert np.array_equal(hecuda.Bfv.inverseNttRows(g, p, out), edge)
    g.close()


def test_relinearize_n32768_mixed_55_and_62_bit():
    n = 32768
    moduli = orc.generate_primes([62, 55, 62, 55], False, n)
    assert {modulus_class(p) for p in moduli} == {NARROW, WIDE}
    t = orc.generate_primes([17], True, 1)[0]
    g, o = hecuda.Context(n, moduli, t), orc.Context(n, moduli, t)
    L = o.L
    _, rk = o.keygen(62)
    key = hecuda.EvaluationKey(g, rk)
    ct3 = orc.fill_uniform(55, moduli[:L], n, 2 * 3 * L).reshape(2, 3, L, n)
    for i in range(L):
        ct3[0, 2, i, :] = moduli[i] - 1
    want = o.relinearize(ct3, rk)
    assert np.array_equal(hecuda.Bfv.relinearize(g, ct3, key), want)
    assert np.array_equal(hecuda.Bfv.relinearizeModSwitchDown(g, ct3, key), o.mod_switch_down(want))
    key.close()
    g.close()
