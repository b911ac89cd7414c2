"""An exact Python-integer model of the library's three lazy sums, and the oracle pinned to it at the accumulators'
bounds (N = 16, 62-bit moduli, operands at p - 1):

- Bfv.innerProduct(ciphertexts:plaintexts:): sum_k ct_k pt_k mod p, reduced every maxLazyProductAccumulationCount
  terms (16 at 62 bits);
- Bfv.innerProduct(_:_:): l0 r0, l0 r1 + l1 r0 and l1 r1 summed over pairs in [Q, Bsk], reduced every
  maxLazyProductAccumulationCount / 2 pairs;
- _computeKeySwitchingUpdate: sum_j digit_j key_j over l digits with one reduction.

The GPU tests in test_gpu_lazy_bounds.py compare the kernels with the oracle at larger N; these checks make sure the
oracle itself is exact where the 128-bit accumulators would overflow without their reductions."""
import numpy as np
import pytest

from oracle import oracle as orc

U128 = 1 << 128


def max_lazy_product_count(qmax, double_bits=128):
    """PolyContext.maxLazyProductAccumulationCount: the most products (qmax - 1)^2 that fit beside qmax."""
    return ((1 << double_bits) - 1 - qmax) // ((qmax - 1) ** 2)


def tensor_sum_cap(pmax):
    """Pairs the device's ct x ct sum accumulates between reductions: every pair adds < 2 p^2 to the middle sum,
    which stays below 2^127."""
    return (1 << 127) // (2 * pmax * pmax)


def ip_plain_model(cts, pts, moduli, present=None):
    """sum_k cts[k] * pts[o][k] mod q_r in Python integers: (terms, polys, l, n) x (rows, terms, l, n) -> the
    (rows, polys, l, n) result and the unreduced (rows, terms, polys, l, n) products."""
    c, p = cts.astype(object), pts.astype(object)
    if present is not None:
        p = p * np.asarray(present, dtype=object)[:, :, None, None]
    prods = c[None, :, :, :, :] * p[:, :, None, :, :]
    q = np.array(moduli, dtype=object)[None, None, :, None]
    return (prods.sum(axis=1) % q).astype(np.uint64), prods


def first_window_sum(prods, window):
    """The largest sum of the first `window` products: what an accumulator holds before its first reduction."""
    return int(prods[:, :window].sum(axis=1).max())


def ct_ct_model(o, lhs, rhs):
    """Bfv.innerProduct(_:_:) with exact tensor sums: lift each operand to [Q, Bsk] and NTT it (the oracle's own,
    separately tested stages), sum the products in Python integers, scale by t, inverse NTT and floor to Q.
    Returns the (groups, 3, L, n) result and the largest unreduced middle sum sum_k (l0 r1 + l1 r0)."""
    n, L = o.n, o.L
    tool = orc.RnsTool(n, o.q, o.t)
    base = o.q + tool.bsk
    R = len(base)
    qb = np.array(base, dtype=object)[:, None]
    groups, pairs = lhs.shape[0], lhs.shape[1]
    out = np.zeros((groups, 3, L, n), dtype=np.uint64)
    widest = 0
    for g in range(groups):
        acc = [np.zeros((R, n), dtype=object) for _ in range(3)]
        for k in range(pairs):
            ev = [orc.ntt_forward(n, base, tool.lift(x)).astype(object)
                  for x in (lhs[g, k, 0], lhs[g, k, 1], rhs[g, k, 0], rhs[g, k, 1])]
            l0, l1, r0, r1 = ev
            acc[0] = acc[0] + l0 * r0
            acc[1] = acc[1] + l0 * r1 + l1 * r0
            acc[2] = acc[2] + l1 * r1
        widest = max(widest, int(acc[1].max()))
        for i in range(3):
            s = ((acc[i] * o.t) % qb).astype(np.uint64)
            out[g, i] = tool.floor(orc.ntt_inverse(n, base, s))
    return out, widest


def ks_digits(n, moduli_ks, target):
    """The key-switching digits dig[r][j] = NTT_{m_r}([target row j]_{m_r}) (Bfv+Keys.swift:165-179)."""
    l = target.shape[0]
    return [[orc.ntt_forward(n, [m], target[j] % np.uint64(m))[0] for j in range(l)] for m in moduli_ks]


def ks_model(o, target, ksk):
    """_computeKeySwitchingUpdate with the digit x key sums in Python integers; returns the (2, l, n) update and the
    largest unreduced sum over rows r, components and columns, with the row's modulus."""
    n, L = o.n, o.L
    l, K = target.shape[0], L + 1
    ksm = o.moduli[:l] + [o.moduli[L]]
    dig = ks_digits(n, ksm, target)
    prod = np.zeros((2, l + 1, n), dtype=np.uint64)
    widest = (0, 1)
    for r, m in enumerate(ksm):
        key_row = K - 1 if r == l else r
        for comp in range(2):
            acc = np.zeros(n, dtype=object)
            for j in range(l):
                acc = acc + dig[r][j].astype(object) * ksk[j, comp, key_row].astype(object)
            top = int(acc.max())
            if top * widest[1] > widest[0] * m:  # compare top / m: the bound crossing is relative to the modulus
                widest = (top, m)
            prod[comp, r] = (acc % m).astype(np.uint64)
    out = np.zeros((2, l, n), dtype=np.uint64)
    for comp in range(2):
        coeff = orc.ntt_inverse(n, ksm, prod[comp])
        out[comp] = orc.divide_round_qlast(n, ksm, coeff)
    return out, widest


def ks_mac_wraps_without_high_reduction(widest):
    """One Montgomery reduction of a < 2^128 returns the high word of a plus up to p: past (2^64 - p) 2^64 that passes
    2^64 (62-bit moduli, l >= 13), unless the high word is first brought below 2p."""
    a, p = widest
    return a >= ((1 << 64) - p) << 64


def ks_mac_reduces_high_word(widest):
    """The key-switching multiply-accumulate subtracts 2p 2^64 from sums whose high word is at least 2p."""
    a, p = widest
    return (a >> 64) >= 2 * p


def constant_target(moduli, l, n, value):
    """l target rows holding `value` in coefficient 0: every digit is `value` at every evaluation point."""
    t = np.zeros((l, n), dtype=np.uint64)
    t[:, 0] = value
    return t


def saturated_key(moduli, L, n):
    """A key-switching key (L, 2, K, N) with every residue m_r - 1: canonical, not a real key."""
    K = L + 1
    key = np.zeros((L, 2, K, n), dtype=np.uint64)
    for r in range(K):
        key[:, :, r, :] = moduli[r] - 1
    return key


N = 16


def test_max_lazy_product_count_at_the_widths():
    """The counts the bounds come from, at the largest primes generate_primes returns."""
    q62 = max(orc.generate_primes([62] * 4, False, N))
    q61 = max(orc.generate_primes([61] * 4, False, N))
    q55 = max(orc.generate_primes([55] * 4, False, N))
    q31 = max(orc.generate_primes([31] * 3, False, N))
    q30 = max(orc.generate_primes([30] * 3, False, N))
    q28 = max(orc.generate_primes([28] * 3, False, N))
    assert max_lazy_product_count(q62) == 16
    assert max_lazy_product_count(q61) == 64
    assert max_lazy_product_count(q55) == 1 << 18
    assert max_lazy_product_count(q31, 64) == 4
    assert max_lazy_product_count(q30, 64) == 16
    assert max_lazy_product_count(q28, 64) == 256


@pytest.mark.parametrize("terms", [15, 16, 17, 32, 33, 48])
@pytest.mark.parametrize("fill", ["max", "uniform"])
def test_oracle_ct_pt_inner_product_at_the_bound(terms, fill):
    moduli = orc.generate_primes([62] * 4, False, N)
    o = orc.Context(N, moduli, 65537)
    L, rows = o.L, 3
    q = moduli[:L]
    if fill == "max":
        cts = np.stack([np.full((terms, 3, N), m - 1, dtype=np.uint64) for m in q], axis=2)
        pts = np.stack([np.full((rows, terms, N), m - 1, dtype=np.uint64) for m in q], axis=2)
    else:
        cts = orc.fill_uniform(terms, q, N, terms * 3 * L).reshape(terms, 3, L, N)
        pts = orc.fill_uniform(terms + 1, q, N, rows * terms * L).reshape(rows, terms, L, N)
    present = np.ones((rows, terms), dtype=np.uint8)
    present[1, 15 % terms] = present[1, 16 % terms] = 0   # nil plaintexts on and next to the reduction point
    present[2, ::2] = 0
    cap = max_lazy_product_count(max(q))
    assert cap == 16
    for pres in (None, present):
        for polys in (1, 2, 3):
            for l in (L, 1):
                c = np.ascontiguousarray(cts[:, :polys, :l])
                p = np.ascontiguousarray(pts[:, :, :l])
                want, prods = ip_plain_model(c, p, q[:l], pres)
                assert np.array_equal(o.inner_product_plain(c, p, pres), want)
                if fill == "max" and pres is None:  # the sum crosses 2^128 exactly when terms > max_terms
                    assert (int(prods.sum(axis=1).max()) >= U128) == (terms > cap)
                    if terms > cap:
                        assert first_window_sum(prods, cap + 1) >= U128


@pytest.mark.parametrize("bits,pairs", [(62, 4), (62, 5), (62, 7), (62, 8), (62, 9), (61, 16), (61, 17), (61, 31)])
def test_oracle_ct_ct_inner_product_at_the_bound(bits, pairs):
    moduli = orc.generate_primes([bits] * 3, False, N)
    o = orc.Context(N, moduli, orc.generate_primes([12], True, 1)[0])
    L = o.L
    groups = 2
    lhs = orc.fill_uniform(bits + pairs, moduli[:L], N, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, N)
    rhs = orc.fill_uniform(bits - pairs, moduli[:L], N, groups * pairs * 2 * L).reshape(groups, pairs, 2, L, N)
    for i in range(L):  # group 0: Q - 1 in coefficient 0 -- every Eval value of every row is its modulus - 1
        lhs[0, :, :, i, :] = 0
        rhs[0, :, :, i, :] = 0
        lhs[0, :, :, i, 0] = moduli[i] - 1
        rhs[0, :, :, i, 0] = moduli[i] - 1
    want, widest = ct_ct_model(o, lhs, rhs)
    assert np.array_equal(o.inner_product(lhs, rhs), want)
    assert widest == pairs * 2 * (max(moduli[:L]) - 1) ** 2  # the Q rows are all at p - 1
    # the device reduces every (2^127 / 2 p_max^2) pairs (4 at 62 bits, 16 at 61): past it the sum crosses 2^127
    assert (widest >= 1 << 127) == (pairs > tensor_sum_cap(max(moduli[:L])))


@pytest.mark.parametrize("l,wraps", [(14, True), (13, True), (12, False)])
def test_oracle_keyswitch_update_at_the_bound(l, wraps):
    moduli = orc.generate_primes([62] * 15, False, N)
    o = orc.Context(N, moduli, 65537)
    L = o.L
    assert L == 14 and len(moduli) == max_lazy_product_count(max(moduli)) - 1  # the most the reference accepts
    key = saturated_key(moduli, L, N)
    target = constant_target(moduli, l, N, min(moduli) - 1)
    want, widest = ks_model(o, target, key)
    assert ks_mac_wraps_without_high_reduction(widest) == wraps
    assert ks_mac_reduces_high_word(widest)
    assert np.array_equal(o.keyswitch_update(target, key), want)
    # a real key: the same model
    _, rk = o.keygen(3)
    target = orc.fill_uniform(l, moduli[:l], N, l)
    want, _ = ks_model(o, target, rk)
    assert np.array_equal(o.keyswitch_update(target, rk), want)
