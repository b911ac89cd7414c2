"""The CPU restatement of the PNNS client (tests/pnns_client_ref.py) pinned on the reference's own tests: ClientTests
(normalizeRowsAndScale, clientConfig, queryAsResponse, clientServer) and UtilsTests (matrixMultiplication,
fixedPointCosineSimilarity)."""
import hashlib

import numpy as np
import pytest

from oracle import client_oracle as co
from oracle import oracle as orc
from oracle import pnns_oracle as opn

import pnns_client_ref as ref


def seed(*parts) -> bytes:
    return hashlib.sha256(repr(parts).encode()).digest()


def test_normalize_rows_and_scale():
    assert ref.normalized_scaled_and_rounded([[3.0, 4.0], [-5.0, 12.0]], 100) == [[60, 80], [-38, 92]]
    assert ref.normalized_scaled_and_rounded([[0.0, 0.0], [1.0, 0.0]], 7) == [[0, 0], [7, 0]]
    with pytest.raises(ValueError):
        ref.normalized_scaled_and_rounded([[np.inf, 1.0]], 7)


def test_matrix_multiplication():
    x = [[-3, -2, -1], [0, 1, 2]]
    y = [[-6, -5, -4, -3], [-2, -1, 0, 1], [2, 3, 4, 5]]
    assert ref.mul_mod(x, y, 100) == [[20, 14, 8, 2], [2, 5, 8, 11]]
    assert ref.mul_mod(x, y, 10) == [[0, 4, -2, 2], [2, -5, -2, 1]]


def test_fixed_point_cosine_similarity():
    x = np.arange(-3, 3, dtype=np.float32).reshape(2, 3)
    y = np.arange(-6, 6, dtype=np.float32).reshape(3, 4)
    xn = x / np.linalg.norm(x, axis=1, keepdims=True)
    yn = y / np.linalg.norm(y, axis=0, keepdims=True)
    expected = xn @ yn
    s = 100
    z = ref.fixed_point_cosine_similarity(x.tolist(), y.tolist(), s * s * 3 + 1, s)
    error = (1 + 1 / (2 * s)) ** 2 - 1          # fixedPointCosineSimilarityError (Util.swift:154-159)
    assert abs(error - 0.010025) < 1e-9
    assert np.all(np.abs(z - expected) <= error)


def test_client_config_max_scaling_factor_grows_with_moduli():
    # PredefinedRlweParameters.n_4096_logq_27_28_28_logt_16 / _logt_17 plaintext moduli
    t16, t17 = 40961, 65537
    one = ref.max_scaling_factor(128, [t16])
    two = ref.max_scaling_factor(128, [t16, t17])
    assert two > one
    assert one == int(np.floor(np.float32(np.sqrt(np.float32((t16 - 1) / 2))) - np.float32(np.sqrt(np.float32(128)) / 2)))


def _context(n, t_bits, q_bits, count=1):
    ts = orc.generate_primes([t_bits] * count, True, n)
    moduli = orc.generate_primes(list(q_bits), False, n)
    return ts, moduli


@pytest.mark.parametrize("extra", [False, True])
def test_query_as_response(extra):
    n, cols, s = 512, 32, 100
    ts, moduli = _context(n, 16, (27, 28, 28))
    if extra:
        ts += orc.generate_primes([17], True, n)
    ctxs = [orc.Context(n, moduli, t) for t in ts]
    sk = co.generate_secret_key(n, moduli, seed("sk", extra))
    query = [[float((1 + c) % ts[0]) for c in range(cols)]]
    count = 1
    a = [[seed("a", k, i) for i in range(count)] for k in range(len(ctxs))]
    e = [[seed("e", k, i) for i in range(count)] for k in range(len(ctxs))]
    cts = ref.generate_query(ctxs, sk, query, s, a, e)
    assert len(cts) == len(ts)
    # a one-row .denseRow matrix reads as a 1 x cols .denseColumn matrix
    got = ref.decrypt(ctxs, sk, [list(c) for c in cts], 1, cols, s)
    scaled = ref.normalized_scaled_and_rounded(query, s)
    assert np.array_equal(got, ref.distances_from_signed(scaled, s))


def client_server(n, ts, moduli, rows, cols, s, ctxs, sk_seed):
    """ClientTests.clientServer for one shape on the restatement: returns (distances, expected)."""
    db = ref.database_for_testing(rows, cols)
    vectors = [v for _, _, v in db]
    query = vectors[:1]
    L = ctxs[0].L
    sk = co.generate_secret_key(n, moduli, sk_seed)
    elements = opn.matrix_evaluation_key_elements(n, rows, cols, 1)
    keys = len(elements) * L
    _, galois = co.generate_evaluation_key(n, moduli[:L], moduli[L], sk, False, elements,
                                           [seed("ka", i) for i in range(keys)], [seed("ke", i) for i in range(keys)])
    values = ref.normalized_scaled_and_rounded(vectors, s)
    flat = [v for row in values for v in row]
    bsgs = opn.BabyStepGiantStep.for_dimension(cols)
    a = [[seed("a", k)] for k in range(len(ctxs))]
    e = [[seed("e", k)] for k in range(len(ctxs))]
    cts = ref.generate_query(ctxs, sk, query, s, a, e)
    replies = []
    for ctx, q in zip(ctxs, cts):
        plain = opn.diagonal_plaintexts(ctx, rows, cols, bsgs, [v % ctx.t for v in flat])
        out = opn.mul_transpose_matrix(ctx, plain, rows, cols, bsgs, list(q), 1, galois)
        replies.append([opn.mod_switch_down_to_single(ctx, ct) for ct in out])
    got = ref.decrypt(ctxs, sk, replies, rows, 1, s)
    modulus = int(np.prod([int(t) for t in ts], dtype=object))
    expected = ref.fixed_point_cosine_similarity(vectors, np.asarray(query, dtype=np.float32).T.tolist(), modulus, s)
    return got, expected


@pytest.mark.parametrize("moduli_count", [1, 2])
@pytest.mark.parametrize("rows", [32, 64, 65, 192])
def test_client_server(rows, moduli_count):
    n, cols = 64, 16
    ts = orc.generate_primes([10] * 2, True, n)[:moduli_count]
    moduli = orc.generate_primes([60] * 3, False, n)
    s = ref.max_scaling_factor(cols, ts)
    ctxs = [orc.Context(n, moduli, t) for t in ts]
    got, expected = client_server(n, ts, moduli, rows, cols, s, ctxs, seed("sk", rows, moduli_count))
    assert got.dtype == np.float32 and got.shape == (rows, 1)
    assert np.array_equal(got, expected)


def test_crt_compose_and_centering():
    moduli = [7, 11, 13]
    for v in range(-500, 500, 37):
        res = [[v % m] for m in moduli]
        assert ref.remainder_to_centered(ref.crt_compose(res, moduli)[0], 7 * 11 * 13) == v


def test_float32_of_int_rounds_ties_to_even():
    assert ref.float32_of_int((1 << 60) + (1 << 36)) == np.float32(2.0 ** 60)           # tie -> even
    assert ref.float32_of_int((1 << 60) + (1 << 36) + 1) == np.float32(2.0 ** 60 + 2.0 ** 37)
    assert ref.float32_of_int(-((1 << 60) + 3 * (1 << 36))) == np.float32(-(2.0 ** 60 + 2.0 ** 38))
