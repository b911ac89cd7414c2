"""Pins of oracle/pnns_oracle.py: SIMD encode/decode round trip, rotation semantics, and the reference's
matrix-multiplication property (MatrixMultiplicationTests: decrypt(M x v^T) == M v mod t)."""
import random

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import pnns_oracle as pn


def context(n=16, t=1153, bits=(55, 52, 62, 58)):
    return orc.Context(n, orc.generate_primes(list(bits), False, n), t)


def test_simd_roundtrip_and_slotwise_product():
    ctx = context()
    rng = random.Random(1)
    a = [rng.randrange(ctx.t) for _ in range(ctx.n)]
    b = [rng.randrange(ctx.t) for _ in range(ctx.n)]
    pa, pb = pn.encode_simd(ctx, a), pn.encode_simd(ctx, b)
    assert pn.decode_simd(ctx, pa).tolist() == a
    prod = orc.ntt_inverse(ctx.n, [ctx.t], orc.poly_op("mul", ctx.n, [ctx.t], orc.ntt_forward(ctx.n, [ctx.t], pa),
                                                       orc.ntt_forward(ctx.n, [ctx.t], pb)))[0]
    assert pn.decode_simd(ctx, prod).tolist() == [x * y % ctx.t for x, y in zip(a, b)]


def test_rotate_columns_moves_simd_slots():
    """HeAPI rotation semantics (HeScheme.swift:960-985): rotateColumns(by: -1) shifts each SIMD row left by one."""
    ctx = context()
    n = ctx.n
    sk, _ = ctx.keygen(3, relin=False)
    values = list(range(1, n + 1))
    ct = ctx.encrypt(4, sk, pn.encode_simd(ctx, values))
    keys = {e: ctx.galois_keygen(50 + e, sk, e) for e in (orc.galois_element_rotating_columns(-1, n),
                                                          orc.galois_element_rotating_columns(2, n))}
    left = pn.decode_simd(ctx, ctx.decrypt(sk, pn.rotate_columns(ctx, ct, -1, keys))).tolist()
    half = n // 2
    assert left == values[1:half] + values[:1] + values[half + 1:] + values[half:half + 1]
    right2 = pn.decode_simd(ctx, ctx.decrypt(sk, pn.rotate_columns(ctx, ct, 2, keys))).tolist()
    assert right2 == values[half - 2:half] + values[:half - 2] + values[n - 2:] + values[half:n - 2]


@pytest.mark.parametrize("n,t,bits,rows,cols", [(16, 1153, (55, 52, 62, 58), 10, 4), (16, 1153, (55, 52, 62, 58), 16, 8),
                                                (16, 1153, (55, 52, 62, 58), 40, 5), (64, 65537, (55, 55, 55), 100, 24),
                                                (64, 65537, (55, 55, 55), 64, 32)])
def test_mul_transpose_vector_is_matrix_vector_product(n, t, bits, rows, cols):
    ctx = context(n, t, bits)
    rng = random.Random(rows * 31 + cols)
    matrix = [[rng.randrange(t) for _ in range(cols)] for _ in range(rows)]
    vector = [rng.randrange(t) for _ in range(cols)]
    bsgs = pn.BabyStepGiantStep.for_dimension(cols)
    plaintexts = pn.diagonal_plaintexts(ctx, rows, cols, bsgs, [v for row in matrix for v in row])
    assert len(plaintexts) == pn.next_power_of_two(cols) * pn.dividing_ceil(rows, n)
    sk, _ = ctx.keygen(9, relin=False)
    keys = {e: ctx.galois_keygen(70 + i, sk, e) for i, e in enumerate(pn.evaluation_key_elements(n, cols))}
    ct = ctx.encrypt(12, sk, pn.dense_row_vector(ctx, vector))
    result = pn.mul_transpose_vector(ctx, plaintexts, rows, bsgs, ct, keys)
    assert len(result) == pn.dividing_ceil(rows, n)
    # the Eval rows converted once give the same ciphertexts (and `plaintexts` is then not read)
    converted = pn.mul_transpose_vector(ctx, None, rows, bsgs, ct, keys, eval_rows=pn.plaintexts_to_eval(ctx, plaintexts))
    assert all(np.array_equal(a, b) for a, b in zip(converted, result)) and len(converted) == len(result)
    expected = [sum(a * b for a, b in zip(row, vector)) % t for row in matrix]
    got = []
    for ct_out in result:
        single = pn.mod_switch_down_to_single(ctx, ct_out)
        got += pn.decode_simd(ctx, ctx.decrypt(sk, single)).tolist()
    assert got[:rows] == expected


def test_baby_step_giant_step_values():
    # BabyStepGiantStep(vectorDimension:) (MatrixMultiplication.swift:55-61)
    for dim, expected in [(1, (1, 1, 1)), (4, (4, 2, 2)), (5, (8, 3, 3)), (128, (128, 12, 11)), (512, (512, 23, 23))]:
        b = pn.BabyStepGiantStep.for_dimension(dim)
        assert (b.vector_dimension, b.baby_step, b.giant_step) == expected


def test_plan_multi_step_examples():
    # GaloisTests.planMultiStep-style: supported {1, 16, 256}: 3 = 1+1+1; 33 = 16+16+1; negative plan when cheaper
    assert pn.plan_multi_step([1, 16, 256], 3, 8192) == {1: 3}
    assert pn.plan_multi_step([1, 16, 256], 33, 8192) == {16: 2, 1: 1}
    assert pn.plan_multi_step([1, 16, 256], 256, 8192) == {256: 1}
    assert pn.plan_multi_step([2, 4], 3, 64) is None
    n = 64
    steps = pn.steps_for([orc.galois_element_rotating_columns(s, n) for s in (1, -1, 4)] + [2 * n - 1], n)
    assert sorted(v for v in steps.values() if v is not None) == [1, 4, n // 2 - 1]
    assert steps[2 * n - 1] is None


@pytest.mark.parametrize("n,t,bits,rows,cols,queries", [
    (16, 1153, (55, 52, 62, 58), 4, 2, 3), (16, 1153, (55, 52, 62, 58), 3, 4, 5), (16, 1153, (55, 52, 62, 58), 8, 4, 2),
    (16, 1153, (55, 52, 62, 58), 20, 3, 3), (64, 65537, (55, 55, 55), 10, 8, 9), (64, 65537, (55, 55, 55), 40, 12, 4),
    (64, 65537, (55, 55, 55), 5, 32, 3)])
def test_mul_transpose_matrix_is_matrix_product(n, t, bits, rows, cols, queries):
    """MatrixMultiplicationTests: (plaintext matrix) x (encrypted query matrix)^T, dense-column packed result."""
    ctx = context(n, t, bits)
    rng = random.Random(rows * 131 + cols * 7 + queries)
    matrix = [[rng.randrange(t) for _ in range(cols)] for _ in range(rows)]
    query = [[rng.randrange(t) for _ in range(cols)] for _ in range(queries)]
    bsgs = pn.BabyStepGiantStep.for_dimension(cols)
    plaintexts = pn.diagonal_plaintexts(ctx, rows, cols, bsgs, [v for row in matrix for v in row])
    sk, _ = ctx.keygen(9, relin=False)
    keys = {e: ctx.galois_keygen(70 + i, sk, e) for i, e in enumerate(pn.matrix_evaluation_key_elements(n, rows, cols, queries))}
    query_plain = pn.dense_row_plaintexts(ctx, queries, cols, [v for row in query for v in row])
    cts = [ctx.encrypt(200 + i, sk, p) for i, p in enumerate(query_plain)]
    result = pn.mul_transpose_matrix(ctx, plaintexts, rows, cols, bsgs, cts, queries, keys)
    decoded = [pn.decode_simd(ctx, ctx.decrypt(sk, pn.mod_switch_down_to_single(ctx, ct))).tolist() for ct in result]
    got = pn.unpack_dense_column(ctx, decoded, rows, queries)
    expected = [sum(a * b for a, b in zip(matrix[r], query[c])) % t for r in range(rows) for c in range(queries)]
    assert got == expected
