"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the PNNS server's matrix-vector product (SURVEY.md 8f rank 3).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.

Reference code followed (paths relative to Sources/):

  * SIMD encoding            HomomorphicEncryption/Encoding.swift:194-246 (generateEncodingMatrix, encodeSimd, decodeSimd)
  * BabyStepGiantStep        PrivateNearestNeighborSearch/MatrixMultiplication.swift:26-62
  * diagonal / dense-row packing   PrivateNearestNeighborSearch/PlaintextMatrix.swift:246-283,341-482
  * mulTranspose(vector:)    MatrixMultiplication.swift:131-226
  * rotateColumnsAndSum      _HomomorphicEncryptionExtras/HeScheme.swift:113-134 (rotations whose key is present)
  * response post-processing Server.swift:61-88 (modSwitchDownToSingle)

Pinned by the property the reference's MatrixMultiplicationTests check: the decrypted, SIMD-decoded result is the
matrix-vector product modulo t (tests/test_oracle_pnns.py).  `mulTranspose(matrix:)` -- extractDenseRow and the
repacking of several result columns into one ciphertext -- is not restated: one dense-row ciphertext per query vector.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from . import oracle as O
from .pir_oracle import dividing_ceil, log2, next_power_of_two

GENERATOR = 3  # GaloisElementGenerator.value (PolyRq/Galois.swift:169-171)


def simd_encoding_matrix(n: int) -> list:
    """HeContext.generateEncodingMatrix (Encoding.swift:196-219)."""
    logn, row, mask = log2(n), n >> 1, 2 * n - 1
    matrix, g = [0] * n, 1
    for i in range(row):
        matrix[i] = O.reverse_bits((g - 1) >> 1, logn)
        matrix[row | i] = O.reverse_bits((mask - g) >> 1, logn)
        g = g * GENERATOR & mask
    return matrix


def encode_simd(ctx: O.Context, values) -> np.ndarray:
    """encodeSimd (Encoding.swift:222-235): scatter into Eval positions, inverse NTT modulo t -> Coeff plaintext."""
    matrix = simd_encoding_matrix(ctx.n)
    ev = np.zeros(ctx.n, dtype=np.uint64)
    for i, v in enumerate(values):
        ev[matrix[i]] = int(v) % ctx.t
    return O.ntt_inverse(ctx.n, [ctx.t], ev)[0]


def decode_simd(ctx: O.Context, plain) -> np.ndarray:
    """decodeSimd (Encoding.swift:237-246)."""
    ev = O.ntt_forward(ctx.n, [ctx.t], np.asarray(plain, dtype=np.uint64))[0]
    return ev[np.array(simd_encoding_matrix(ctx.n))]


@dataclass(frozen=True)
class BabyStepGiantStep:
    """BabyStepGiantStep (MatrixMultiplication.swift:26-62)."""

    vector_dimension: int
    baby_step: int
    giant_step: int

    @staticmethod
    def for_dimension(vector_dimension: int) -> "BabyStepGiantStep":
        dimension = next_power_of_two(vector_dimension)
        baby = math.isqrt(dimension)
        if baby * baby < dimension:
            baby += 1  # Int(Double(dimension).squareRoot().rounded(.up))
        giant = dividing_ceil(dimension, baby)
        assert baby >= giant
        return BabyStepGiantStep(dimension, baby, giant)


def evaluation_key_elements(n: int, column_count: int) -> list:
    """The rotations mulTranspose(vector:) needs (MatrixMultiplication.swift:84-94): by -1 and by -babyStep."""
    bsgs = BabyStepGiantStep.for_dimension(column_count)
    return [O.galois_element_rotating_columns(-1, n), O.galois_element_rotating_columns(-bsgs.baby_step, n)]


def diagonal_plaintexts(ctx: O.Context, row_count: int, column_count: int, bsgs: BabyStepGiantStep, values) -> list:
    """PlaintextMatrix.diagonalPlaintexts (PlaintextMatrix.swift:417-482) -> Coeff plaintexts."""
    n = ctx.n
    assert column_count <= n // 2
    data = np.asarray(values, dtype=np.uint64).reshape(row_count, column_count)
    padded_rows = next_power_of_two(column_count)
    packed = np.zeros((padded_rows, row_count), dtype=np.uint64)
    for r in range(padded_rows):
        for c in range(row_count):
            pc = (c + r) % padded_rows
            if pc < column_count:
                packed[r, c] = data[c, pc]
    per_column = dividing_ceil(row_count, n)
    out = []
    for r in range(padded_rows):
        for chunk_index in range(per_column):
            chunk = np.zeros(n, dtype=np.uint64)
            piece = packed[r, chunk_index * n:(chunk_index + 1) * n]
            chunk[: len(piece)] = piece
            i = (len(out) - chunk_index) // per_column
            step = (i // bsgs.baby_step) * bsgs.baby_step
            if step:
                half = n // 2
                chunk = np.concatenate([np.roll(chunk[:half], step), np.roll(chunk[half:], step)])
            out.append(encode_simd(ctx, chunk))
    assert len(out) == padded_rows * per_column
    return out


def dense_row_vector(ctx: O.Context, vector) -> np.ndarray:
    """PlaintextMatrix.denseRowPlaintexts for ONE row (PlaintextMatrix.swift:341-413): the row, padded to a power of
    two, repeated to fill both SIMD rows."""
    n = ctx.n
    v = [int(x) % ctx.t for x in vector]
    packed = v + [0] * (next_power_of_two(len(v)) - len(v))
    simd_columns = n // 2
    if len(packed) < simd_columns and len(packed) + len(v) > simd_columns:
        packed += [0] * (simd_columns - len(packed))
    offset = len(packed) % simd_columns
    packed += [0] * (0 if offset == 0 else next_power_of_two(offset) - offset)
    repeat = list(packed) if len(packed) <= simd_columns else packed[simd_columns:]
    while len(packed) < n:
        packed += repeat
    return encode_simd(ctx, packed)


def _add(ctx, a, b):
    l = a.shape[-2]
    q = np.array(ctx.q[:l], dtype=np.uint64)[None, :, None]
    return (a + b) % q


def rotate_columns(ctx, ct, step: int, galois_keys: dict):
    """Bfv.rotateColumns (HeScheme.swift:1463-1470) = applyGalois with GaloisElement.rotatingColumns(by:degree:)."""
    element = O.galois_element_rotating_columns(step, ctx.n)
    if element not in galois_keys:
        raise KeyError("missingGaloisElement")
    return ctx.apply_galois(ct, element, galois_keys[element], threads=1)[0]


def rotate_columns_and_sum(ctx, cts: list, step: int, galois_keys: dict):
    """HeScheme.rotateColumnsAndSum (_HomomorphicEncryptionExtras/HeScheme.swift:113-134)."""
    cts = list(cts)
    acc = cts.pop()
    for ct in reversed(cts):
        acc = rotate_columns(ctx, acc, step, galois_keys)
        acc = _add(ctx, acc, ct)
    return acc


def plaintexts_to_eval(ctx: O.Context, plaintexts: list, l: int = 0) -> np.ndarray:
    """The diagonal packing's Coeff plaintexts in Eval format over the first l moduli: (count, l, N)."""
    return np.stack([ctx.plaintext_to_eval(p, l) for p in plaintexts])


def mul_transpose_vector(ctx: O.Context, plaintexts: list, row_count: int, bsgs: BabyStepGiantStep, ct, galois_keys: dict,
                         eval_rows=None):
    """PlaintextMatrix.mulTranspose(vector:using:) (MatrixMultiplication.swift:131-226).  plaintexts: the diagonal
    packing in Coeff format; ct: dense-row ciphertext (2, L, N) Coeff.  Returns resultCiphertextCount ciphertexts.
    eval_rows: optionally the same plaintexts already in Eval format over the ciphertext's moduli (plaintexts_to_eval),
    so that many calls over one matrix convert it once; `plaintexts` is then not read."""
    n, L = ctx.n, ct.shape[-2]
    if eval_rows is not None:
        assert eval_rows.shape[1:] == (L, n)
    states, state = [], ct
    for step in range(bsgs.baby_step):
        states.append(state)
        if step != bsgs.baby_step - 1:
            state = rotate_columns(ctx, state, -1, galois_keys)
    rotated = np.stack([np.stack([O.ntt_forward(n, ctx.q[:L], s[p]) for p in range(2)]) for s in states])
    result_count = dividing_ceil(row_count, n)
    out = []
    for r in range(result_count):
        to_add = []
        for g in range(bsgs.giant_step):
            count = min(len(states), bsgs.vector_dimension - bsgs.baby_step * g)
            indices = [result_count * (j + bsgs.baby_step * g) + r for j in range(count)]
            if eval_rows is None:
                rows = np.stack([ctx.plaintext_to_eval(plaintexts[i], L) for i in indices])
            else:
                rows = eval_rows[indices]
            ip = ctx.inner_product_plain(rotated[:count], rows[None], None, threads=1)[0]
            to_add.append(np.stack([O.ntt_inverse(n, ctx.q[:L], ip[p]) for p in range(2)]))
        out.append(rotate_columns_and_sum(ctx, to_add, -bsgs.baby_step, galois_keys))
    return out


def mod_switch_down_to_single(ctx, ct):
    while ct.shape[-2] > 1:
        ct = ctx.mod_switch_down(ct, threads=1)[0]
    return ct


# ------------------------------------------------------------------------------------------------ matrix path
def dense_row_plaintexts(ctx: O.Context, row_count: int, column_count: int, values) -> list:
    """PlaintextMatrix.denseRowPlaintexts (PlaintextMatrix.swift:341-413) for any number of rows -> Coeff plaintexts."""
    n, simd_columns = ctx.n, ctx.n // 2
    assert column_count <= simd_columns
    vals = [int(v) % ctx.t for v in values]
    pad = [0] * (next_power_of_two(column_count) - column_count)
    out, packed, idx = [], [], 0
    for _ in range(row_count):
        packed += vals[idx:idx + column_count] + pad
        idx += column_count
        if len(packed) < simd_columns and len(packed) + column_count > simd_columns:
            packed += [0] * (simd_columns - len(packed))
        if len(packed) + column_count > n:
            out.append(encode_simd(ctx, packed))
            packed = []
    if packed:
        offset = len(packed) % simd_columns
        packed += [0] * (0 if offset == 0 else next_power_of_two(offset) - offset)
        repeat = list(packed) if len(packed) <= simd_columns else packed[simd_columns:]
        while len(packed) < n:
            packed += repeat
        out.append(encode_simd(ctx, packed[:n]))
    rows_per_plaintext = 2 * (simd_columns // next_power_of_two(column_count))
    assert len(out) == dividing_ceil(row_count, rows_per_plaintext)
    return out


def steps_for(elements: list, degree: int) -> dict:
    """GaloisElement.stepsFor (PolyRq/Galois.swift:239-258): element 3^k <-> rotation step N/2 - k."""
    result = {e: None for e in elements}
    found, g = 0, 1
    for step in range(degree // 2 + 1):
        if g in result and result[g] is None:
            result[g] = degree // 2 - step
            found += 1
            if found == len(result):
                break
        g = g * GENERATOR % (2 * degree)
    return result


def _plan_greedy(sorted_steps, step, transform):
    plan, remaining = {}, transform(step)
    for s in sorted_steps:
        ts = transform(s)
        count = remaining // ts
        if count > 0:
            plan[s] = plan.get(s, 0) + count
        remaining %= ts
    return plan if remaining == 0 else None


def plan_multi_step(supported_steps: list, step: int, degree: int):
    """GaloisElement._planMultiStep (PolyRq/Galois.swift:272-319)."""
    assert abs(step) < degree
    if step in supported_steps:
        return {step: 1}
    descending = sorted(supported_steps, reverse=True)
    positive = _plan_greedy(descending, step, lambda s: s)
    negative = _plan_greedy(list(reversed(descending)), step, lambda s: (degree >> 1) - s)
    if positive is None or negative is None:
        return positive if negative is None else negative
    return positive if sum(positive.values()) <= sum(negative.values()) else negative


def rotation_sequence(galois_elements: list, step: int, degree: int) -> list:
    """The single rotations rotateColumnsMultiStep performs (_HomomorphicEncryptionExtras/HeScheme.swift:65-104).
    The reference iterates a Swift Dictionary, whose order is unspecified; here: larger steps first."""
    if step == 0:
        return []
    if O.galois_element_rotating_columns(step, degree) in galois_elements:
        return [step]
    steps = [s for s in steps_for(list(galois_elements), degree).values() if s is not None]
    positive = step + degree // 2 if step < 0 else step
    plan = plan_multi_step(steps, positive, degree)
    if plan is None:
        raise ValueError("invalidRotationStep")
    return [s for s in sorted(plan, reverse=True) for _ in range(plan[s])]


def rotate_columns_multi_step(ctx, ct, step: int, galois_keys: dict):
    for s in rotation_sequence(list(galois_keys), step, ctx.n):
        ct = rotate_columns(ctx, ct, s, galois_keys)
    return ct


def rotate_columns_multi_step_and_sum(ctx, cts: list, step: int, galois_keys: dict):
    """rotateColumnsAndSum with rotateColumnsMultiStep (_HomomorphicEncryptionExtras/HeScheme.swift:113-134)."""
    cts = list(cts)
    acc = cts.pop()
    for ct in reversed(cts):
        acc = rotate_columns_multi_step(ctx, acc, step, galois_keys)
        acc = _add(ctx, acc, ct)
    return acc


def swap_rows(ctx, ct, galois_keys: dict):
    element = O.galois_element_swapping_rows(ctx.n)
    return ctx.apply_galois(ct, element, galois_keys[element], threads=1)[0]


@dataclass
class DenseRowExtraction:
    """What extractDenseRow does for one row (CiphertextMatrix.swift:245-352), as data."""

    ciphertext_index: int
    mask: list            # SIMD values of the plaintext mask
    rotate_count: int
    column_step: int      # columnCount.nextPowerOfTwo


def dense_row_extraction(n: int, row_count: int, column_count: int, ciphertext_count: int, row_index: int) -> DenseRowExtraction:
    simd_columns = n // 2
    cpow = next_power_of_two(column_count)
    rows_per_ciphertext = 2 * (simd_columns // cpow)
    ciphertext_index = row_index // rows_per_ciphertext

    def slot_range(r):
        start = (r % rows_per_ciphertext) * cpow
        lo, hi = start, start + cpow
        if lo <= simd_columns < hi:
            lo, hi = simd_columns, simd_columns + cpow
        elif hi > simd_columns:
            padding = simd_columns % cpow
            lo, hi = lo + padding, hi + padding
        if ciphertext_index == ciphertext_count - 1:
            hi = dividing_ceil(hi, simd_columns) * simd_columns
        return lo, hi

    lo, hi = slot_range(row_index)
    last = row_index + 1
    while last < row_count and slot_range(last)[1] == hi:
        last += 1
    first = row_index - 1 if row_index > 0 else 0
    while first > 0 and slot_range(first)[1] == hi:
        first -= 1
    rows_in_batch = last - first
    repeat = [1] * cpow + [0] * (cpow * (rows_in_batch - 1))
    repeat += [0] * (next_power_of_two(len(repeat)) - len(repeat))
    mask, copies = [0] * lo, 0
    while len(mask) < hi:
        mask += repeat
        copies += 1
    mask = mask[:n]
    return DenseRowExtraction(ciphertext_index, mask, simd_columns // (copies * cpow) - 1, cpow)


def extract_dense_row(ctx, ciphertexts: list, row_count: int, column_count: int, row_index: int, galois_keys: dict):
    """CiphertextMatrix.extractDenseRow (CiphertextMatrix.swift:245-352)."""
    if row_count == 1:
        return ciphertexts[0]
    n = ctx.n
    ex = dense_row_extraction(n, row_count, column_count, len(ciphertexts), row_index)
    ct = ciphertexts[ex.ciphertext_index]
    L = ct.shape[-2]
    ev = np.stack([O.ntt_forward(n, ctx.q[:L], ct[p]) for p in range(2)])
    mask_eval = ctx.plaintext_to_eval(encode_simd(ctx, ex.mask), L)
    prod = ctx.inner_product_plain(ev[None], mask_eval[None, None], None, threads=1)[0]   # ciphertextEval *= plaintextMask
    ct = np.stack([O.ntt_inverse(n, ctx.q[:L], prod[p]) for p in range(2)])
    copy_right = ct
    for _ in range(ex.rotate_count):
        copy_right = rotate_columns(ctx, copy_right, ex.column_step, galois_keys)
        ct = _add(ctx, ct, copy_right)
    return _add(ctx, ct, swap_rows(ctx, ct, galois_keys))


def matrix_evaluation_key_elements(n: int, matrix_rows: int, matrix_columns: int, max_query_count: int) -> list:
    """MatrixMultiplication.evaluationKeyConfig (MatrixMultiplication.swift:76-116) + extractDenseRowConfig
    (CiphertextMatrix.swift:224-243)."""
    simd_columns = n // 2
    bsgs = BabyStepGiantStep.for_dimension(matrix_columns)
    rot = O.galois_element_rotating_columns
    elements = [rot(-1, n), rot(-bsgs.baby_step, n), O.galois_element_swapping_rows(n)]
    if simd_columns // matrix_rows > 1:
        elements.append(rot(1, n))
        if simd_columns > 16:
            elements.append(rot(16, n))
        if simd_columns > 256:
            elements.append(rot(256, n))
    if max_query_count != 1:
        cpow = next_power_of_two(matrix_columns)
        if cpow != simd_columns:
            elements.append(rot(cpow, n))
    return list(dict.fromkeys(elements))


def mul_transpose_matrix(ctx, plaintexts: list, matrix_rows: int, matrix_columns: int, bsgs: BabyStepGiantStep,
                         ciphertexts: list, query_rows: int, galois_keys: dict) -> list:
    """PlaintextMatrix.mulTranspose(matrix:using:) (MatrixMultiplication.swift:236-298): dense-column packed result."""
    n, simd_columns = ctx.n, ctx.n // 2
    inner = []
    for row in range(query_rows):
        ct = extract_dense_row(ctx, ciphertexts, query_rows, matrix_columns, row, galois_keys)
        inner += mul_transpose_vector(ctx, plaintexts, matrix_rows, bsgs, ct, galois_keys)
    per_simd_row = simd_columns // matrix_rows
    if per_simd_row > 0:
        per_ciphertext = 2 * per_simd_row
        packed = []
        for start in range(0, len(inner), per_ciphertext):
            chunk = inner[start:start + per_ciphertext]
            rows = [rotate_columns_multi_step_and_sum(ctx, chunk[s:s + per_simd_row], matrix_rows, galois_keys)
                    for s in range(0, len(chunk), per_simd_row)]
            if len(chunk) > per_simd_row:   # swapRowsAndAdd(swapping: packedRows[1], addingTo: packedRows[0])
                packed.append(_add(ctx, swap_rows(ctx, rows[1], galois_keys), rows[0]))
            else:
                packed.append(rows[0])
        inner = packed
    return inner


def unpack_dense_column(ctx, decoded: list, row_count: int, column_count: int) -> list:
    """PlaintextMatrix.unpackDenseColumn (PlaintextMatrix.swift:515-556): SIMD-decoded plaintexts -> row-major values."""
    simd_columns = ctx.n // 2
    per_plaintext = 2 * (simd_columns // row_count)
    total = row_count * column_count
    column_major = []
    for d in decoded:
        d = list(d)
        if per_plaintext > 1:
            per_simd_row = row_count * (simd_columns // row_count)
            take = min(per_simd_row, total - len(column_major))
            column_major += d[:take]
            take = min(per_simd_row, total - len(column_major))
            column_major += d[simd_columns:simd_columns + take]
        else:
            in_row = len(column_major) % row_count
            column_major += d[:min(len(d), row_count - in_row)]
    assert len(column_major) == total
    return [column_major[c * row_count + r] for r in range(row_count) for c in range(column_count)]
