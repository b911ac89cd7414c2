"""hecuda.pnns -- host-side mirror of the PNNS server's matrix-vector product over libhecuda (SURVEY.md 8f rank 3).

    BabyStepGiantStep, MatrixDimensions        PrivateNearestNeighborSearch/MatrixMultiplication.swift:26-62,
                                               PlaintextMatrix.swift:45-72
    PlaintextMatrix (.diagonal packing)        PlaintextMatrix.swift:417-482
    PlaintextMatrix.mulTranspose(vector:using:) MatrixMultiplication.swift:131-226
    SIMD encoding                              HomomorphicEncryption/Encoding.swift:194-246

The diagonal packing and the SIMD encoding of the database are host work in the reference too (offline
preprocessing); conversion to Eval format, the rotations, inner products and modulus switching run on the device.
`mulTransposeMatrix` runs the whole mulTranspose(matrix:) -- extractDenseRow, products, dense-column packing -- in one
C-ABI call; the shape logic extractDenseRow derives per row (mask, ciphertext index, replication count) is computed here.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Any

import numpy as np

from . import Context, EvaluationKey, HeError, _check, _host, _ptr, load_library


class PnnsError(ValueError):
    pass


def _next_power_of_two(v: int) -> int:
    return 1 << max(0, (int(v) - 1).bit_length())


@dataclass(frozen=True)
class BabyStepGiantStep:
    """BabyStepGiantStep (MatrixMultiplication.swift:26-62)."""

    vectorDimension: int
    babyStep: int
    giantStep: int

    def __post_init__(self):
        if self.babyStep < self.giantStep:
            raise PnnsError("babyStep cannot be smaller than giantStep")

    @staticmethod
    def forVectorDimension(vectorDimension: int) -> "BabyStepGiantStep":
        dimension = _next_power_of_two(vectorDimension)
        baby = math.isqrt(dimension - 1) + 1 if dimension > 1 else 1   # ceil(sqrt(dimension))
        return BabyStepGiantStep(dimension, baby, -(-dimension // baby))


@dataclass(frozen=True)
class MatrixDimensions:
    """MatrixDimensions (PlaintextMatrix.swift:45-72)."""

    rowCount: int
    columnCount: int

    def __post_init__(self):
        if self.rowCount <= 0 or self.columnCount <= 0:
            raise PnnsError(f"invalidMatrixDimensions(rowCount: {self.rowCount}, columnCount: {self.columnCount})")


class GaloisElement:
    """GaloisElement.rotatingColumns / swappingRows (PolyRq/Galois.swift:174-212)."""

    @staticmethod
    def rotatingColumns(step: int, degree: int) -> int:
        positive = abs(step)
        if not 0 < positive < degree >> 1:
            raise HeError(-1, f"invalidRotationStep(step: {step}, degree: {degree})")
        if step > 0:
            positive = (degree >> 1) - positive
        return pow(3, positive, 2 * degree)

    @staticmethod
    def swappingRows(degree: int) -> int:
        return 2 * degree - 1

    @staticmethod
    def stepsFor(elements, degree: int) -> dict:
        """GaloisElement.stepsFor (PolyRq/Galois.swift:239-258): 3^k mod 2N  <->  rotation by N/2 - k."""
        wanted, out, g = set(int(e) for e in elements), {}, 1
        for k in range(degree // 2 + 1):
            if g in wanted and g not in out:
                out[g] = degree // 2 - k
            g = g * 3 % (2 * degree)
        return {e: out.get(e) for e in wanted}

    @staticmethod
    def planMultiStep(supportedSteps, step: int, degree: int):
        """GaloisElement._planMultiStep (PolyRq/Galois.swift:272-319): greedy decomposition, by steps or by their
        complements to N/2, whichever needs fewer rotations."""
        if abs(step) >= degree:
            raise HeError(-1, f"invalidRotationStep(step: {step}, degree: {degree})")
        if step in supportedSteps:
            return {step: 1}

        def greedy(order, weight):
            left, plan = weight(step), {}
            for s in order:
                w = weight(s)
                if left // w:
                    plan[s] = plan.get(s, 0) + left // w
                left %= w
            return plan if left == 0 else None

        down = sorted(supportedSteps, reverse=True)
        forward = greedy(down, lambda s: s)
        backward = greedy(down[::-1], lambda s: (degree >> 1) - s)
        if forward is None or backward is None:
            return forward if backward is None else backward
        return forward if sum(forward.values()) <= sum(backward.values()) else backward

    @staticmethod
    def rotationSequence(galoisElements, step: int, degree: int) -> list:
        """The single rotations of rotateColumnsMultiStep(by: step) (_HomomorphicEncryptionExtras/HeScheme.swift:65-104),
        larger steps first (the reference walks a Dictionary, i.e. in unspecified order)."""
        if step == 0:
            return []
        if GaloisElement.rotatingColumns(step, degree) in galoisElements:
            return [step]
        steps = [s for s in GaloisElement.stepsFor(galoisElements, degree).values() if s is not None]
        plan = GaloisElement.planMultiStep(steps, step + degree // 2 if step < 0 else step, degree)
        if plan is None:
            raise HeError(-1, f"invalidRotationStep(step: {step}, degree: {degree})")
        return [s for s in sorted(plan, reverse=True) for _ in range(plan[s])]


class CiphertextMatrix:
    """The shape logic of CiphertextMatrix in `.denseRow` packing (CiphertextMatrix.swift, PlaintextMatrix.swift:262-268)."""

    @staticmethod
    def ciphertextCount(degree: int, dimensions: MatrixDimensions) -> int:
        per_ciphertext = 2 * ((degree // 2) // _next_power_of_two(dimensions.columnCount))
        return -(-dimensions.rowCount // per_ciphertext)

    @staticmethod
    def denseRowExtraction(degree: int, dimensions: MatrixDimensions, ciphertextCount: int, rowIndex: int):
        """What extractDenseRow derives for one row (CiphertextMatrix.swift:254-320): (index of the ciphertext holding
        the row, SIMD values of the plaintext mask, number of rotate-and-add replication steps)."""
        columns = degree // 2
        width = _next_power_of_two(dimensions.columnCount)
        per_ciphertext = 2 * (columns // width)
        ciphertext_index = rowIndex // per_ciphertext
        is_last = ciphertext_index == ciphertextCount - 1

        def slots(row):
            lo = (row % per_ciphertext) * width
            hi = lo + width
            if lo <= columns < hi:                       # the batch would straddle the two SIMD rows
                lo, hi = columns, columns + width
            elif hi > columns:                           # second SIMD row: skip the first row's padding
                lo, hi = lo + columns % width, hi + columns % width
            if is_last:                                  # the last ciphertext repeats its rows to the end
                hi = -(-hi // columns) * columns
            return lo, hi

        lo, hi = slots(rowIndex)
        after = rowIndex + 1
        while after < dimensions.rowCount and slots(after)[1] == hi:
            after += 1
        before = max(rowIndex - 1, 0)
        while before > 0 and slots(before)[1] == hi:
            before -= 1
        period = _next_power_of_two(width * (after - before))
        mask = [0] * lo
        copies = 0
        while len(mask) < hi:
            mask += [1] * width + [0] * (period - width)
            copies += 1
        return ciphertext_index, mask[:degree], columns // (copies * width) - 1


class SimdEncoder:
    """Context.encode(values:format: .simd) / decode (Encoding.swift:194-246) for a plaintext modulus t = 1 mod 2N,
    with the reference's choice of the minimal primitive 2N-th root of unity (PolyContext / NTT tables)."""

    def __init__(self, degree: int, plaintextModulus: int):
        n, t = int(degree), int(plaintextModulus)
        if (t - 1) % (2 * n) or t >= 1 << 32:
            raise HeError(-2, "simdEncodingNotSupported: t must be an NTT-friendly prime below 2^32")
        self.n, self.t, self.logn = n, t, n.bit_length() - 1
        self.psi = self._minimal_root()
        rev = self._bit_reverse(np.arange(n), self.logn)
        powers = np.ones(n, dtype=np.uint64)
        for i in range(1, n):
            powers[i] = int(powers[i - 1]) * self.psi % t
        self.roots = powers[rev]                                   # psi^bitrev(i), the merged-twiddle table
        inverse = pow(self.psi, -1, t)
        ipowers = np.ones(n, dtype=np.uint64)
        for i in range(1, n):
            ipowers[i] = int(ipowers[i - 1]) * inverse % t
        self.inverse_roots = ipowers[rev]
        half, mask = n >> 1, 2 * n - 1
        g, matrix = 1, np.zeros(n, dtype=np.int64)
        for i in range(half):
            matrix[i] = self._bit_reverse(np.array([(g - 1) >> 1]), self.logn)[0]
            matrix[half | i] = self._bit_reverse(np.array([(mask - g) >> 1]), self.logn)[0]
            g = g * 3 & mask
        self.encodingMatrix = matrix

    @staticmethod
    def _bit_reverse(x, bits):
        x = np.asarray(x, dtype=np.int64)
        out = np.zeros_like(x)
        for b in range(bits):
            out |= ((x >> b) & 1) << (bits - 1 - b)
        return out

    def _minimal_root(self) -> int:
        n, t = self.n, self.t
        root = next(r for r in (pow(x, (t - 1) // (2 * n), t) for x in range(2, t)) if pow(r, n, t) == t - 1)
        best, cur, sq = root, root, root * root % t
        for _ in range(n - 1):          # all primitive 2N-th roots are the odd powers of one of them
            cur = cur * sq % t
            best = min(best, cur)
        return best

    def forwardNtt(self, coeffs: np.ndarray) -> np.ndarray:
        """rows x N, natural order in -> bit-reversed Eval out (same convention as PolyRq.forwardNtt)."""
        a = np.array(coeffs, dtype=np.uint64).reshape(-1, self.n)
        t = np.uint64(self.t)
        m, span = 1, self.n >> 1
        while m < self.n:
            a = a.reshape(a.shape[0], m, 2, span)
            w = self.roots[m:2 * m].reshape(1, m, 1)
            v = a[:, :, 1, :] * w % t
            u = a[:, :, 0, :]
            a = np.stack([(u + v) % t, (u + t - v) % t], axis=2)
            m, span = m * 2, span >> 1
        return a.reshape(-1, self.n)

    def inverseNtt(self, evals: np.ndarray) -> np.ndarray:
        a = np.array(evals, dtype=np.uint64).reshape(-1, self.n)
        t = np.uint64(self.t)
        m, span = self.n >> 1, 1
        while m >= 1:
            a = a.reshape(a.shape[0], m, 2, span)
            w = self.inverse_roots[m:2 * m].reshape(1, m, 1)
            u, v = a[:, :, 0, :], a[:, :, 1, :]
            a = np.stack([(u + v) % t, (u + t - v) % t * w % t], axis=2)
            m, span = m >> 1, span * 2
        return a.reshape(-1, self.n) * np.uint64(pow(self.n, -1, self.t)) % t

    def encode(self, values: np.ndarray) -> np.ndarray:
        """rows x (<= N) SIMD values -> rows x N coefficient plaintexts."""
        v = np.asarray(values, dtype=np.uint64)
        v = v.reshape(-1, v.shape[-1])
        ev = np.zeros((v.shape[0], self.n), dtype=np.uint64)
        ev[:, self.encodingMatrix[: v.shape[1]]] = v % np.uint64(self.t)
        return self.inverseNtt(ev)

    def decode(self, plaintexts: np.ndarray) -> np.ndarray:
        return self.forwardNtt(plaintexts)[:, self.encodingMatrix]


def _signed(values, dimensions: MatrixDimensions) -> np.ndarray:
    v = np.ascontiguousarray(np.asarray(values, dtype=np.int64)).reshape(-1)
    if v.size != dimensions.rowCount * dimensions.columnCount:
        raise PnnsError(f"wrongValueCount(got: {v.size}, expected: {dimensions.rowCount * dimensions.columnCount})")
    return v


def centeredToRemainder(values, modulus: int) -> np.ndarray:
    """Scalar.centeredToRemainder (ModularArithmetic/Scalar.swift:85-95): x in [-floor(t/2), floor((t-1)/2)] -> x mod t."""
    v = np.asarray(values, dtype=np.int64)
    if v.size and (int(v.max()) > (modulus - 1) // 2 or int(v.min()) < -(modulus // 2)):
        raise PnnsError("centeredToRemainder: value outside [-floor(t/2), floor((t-1)/2)]")
    return np.where(v < 0, v + modulus, v).astype(np.uint64)


class PlaintextMatrix:
    """PlaintextMatrix<Bfv<UInt64>, Eval> in .diagonal packing, resident in HBM."""

    def __init__(self, context: Context, dimensions: MatrixDimensions, values, babyStepGiantStep: BabyStepGiantStep = None,
                 plaintexts=None, evalFormat: bool = False):
        """values: the matrix in row-major order (packed here), or plaintexts: the already packed diagonal plaintexts
        (count x N coefficient rows, or count x L x N with evalFormat) as PlaintextMatrix.init(dimensions:packing:plaintexts:)."""
        self.context, self.dimensions = context, dimensions
        self.babyStepGiantStep = babyStepGiantStep or BabyStepGiantStep.forVectorDimension(dimensions.columnCount)
        if plaintexts is None:
            rows = PlaintextMatrix.diagonalPlaintexts(context, dimensions, self.babyStepGiantStep, values)
        else:
            rows = _host(plaintexts)
            expected = self.babyStepGiantStep.vectorDimension * -(-dimensions.rowCount // context.degree)
            if rows.size != expected * context.degree * (context.L if evalFormat else 1):
                raise PnnsError(f"wrongPlaintextCount(got: {rows.size // context.degree}, expected: {expected})")
        h = C.c_void_p()
        _check(load_library().hecuda_pnns_matrix_create(context._h, _ptr(rows), 1 if evalFormat else 0, dimensions.rowCount, dimensions.columnCount,
                                                       self.babyStepGiantStep.babyStep, self.babyStepGiantStep.giantStep,
                                                       C.byref(h)))
        self._h = h
        self.resultCiphertextCount = -(-dimensions.rowCount // context.degree)

    @classmethod
    def fromSignedValues(cls, context: Context, dimensions: MatrixDimensions, signedValues,
                         babyStepGiantStep: BabyStepGiantStep = None, reduce: bool = False) -> "PlaintextMatrix":
        """PlaintextMatrix.init(context:dimensions:packing: .diagonal, signedValues:reduce:) (PlaintextMatrix.swift:155-190)
        followed by convertToEvalFormat, all on the device (hecuda_pnns_matrix_create_from_values): only the values
        cross PCIe.  The resident words equal those of `PlaintextMatrix(context, dimensions, v)` with each value v
        mapped by centeredToRemainder (or reduced mod t with `reduce`)."""
        bsgs = babyStepGiantStep or BabyStepGiantStep.forVectorDimension(dimensions.columnCount)
        values = _signed(signedValues, dimensions)
        h = C.c_void_p()
        _check(load_library().hecuda_pnns_matrix_create_from_values(
            context._h, _ptr(values), 1 if reduce else 0, dimensions.rowCount, dimensions.columnCount, bsgs.babyStep,
            bsgs.giantStep, C.byref(h)))
        m = cls.__new__(cls)
        m.context, m.dimensions, m.babyStepGiantStep, m._h = context, dimensions, bsgs, h
        m.resultCiphertextCount = -(-dimensions.rowCount // context.degree)
        return m

    @staticmethod
    def diagonalPlaintextsOnDevice(context: Context, dimensions: MatrixDimensions, bsgs: BabyStepGiantStep, signedValues,
                                   reduce: bool = False) -> np.ndarray:
        """diagonalPlaintexts of signed values on the device (hecuda_pnns_diagonal_plaintexts): count x N coefficient
        rows, equal to `diagonalPlaintexts(context, dimensions, bsgs, centeredToRemainder(signedValues))`."""
        values = _signed(signedValues, dimensions)
        count = _next_power_of_two(dimensions.columnCount) * -(-dimensions.rowCount // context.degree)
        out = np.empty((count, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_pnns_diagonal_plaintexts(context._h, _ptr(values), 1 if reduce else 0,
                                                              dimensions.rowCount, dimensions.columnCount, bsgs.babyStep,
                                                              _ptr(out)))
        return out

    def deviceBuffer(self):
        """(device pointer, bytes) of the resident [result][giant][baby] x L x N Eval words."""
        p, n = C.c_void_p(), C.c_uint64(0)
        _check(load_library().hecuda_pnns_matrix_device_buffer(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def presentFlags(self) -> np.ndarray:
        """The resident presence flags in [result][giant][baby] slot order: 0 for an absent plaintext."""
        count = self.resultCiphertextCount * self.babyStepGiantStep.giantStep * self.babyStepGiantStep.babyStep
        out = np.empty(count, dtype=np.uint8)
        _check(load_library().hecuda_pnns_matrix_present(self._h, _ptr(out), count))
        return out

    @staticmethod
    def diagonalPlaintexts(context, dimensions: MatrixDimensions, bsgs: BabyStepGiantStep, values) -> np.ndarray:
        """PlaintextMatrix.diagonalPlaintexts (PlaintextMatrix.swift:417-482) as coefficient rows (count x N).
        `context` only needs `degree` and `plaintextModulus`."""
        n, t = context.degree, context.plaintextModulus
        rows, cols = dimensions.rowCount, dimensions.columnCount
        if cols > n // 2:
            raise PnnsError(f"invalidMatrixDimensions(rowCount: {rows}, columnCount: {cols})")
        data = np.asarray(values, dtype=np.uint64).reshape(rows, cols)
        padded = _next_power_of_two(cols)
        wide = np.zeros((rows, padded), dtype=np.uint64)
        wide[:, :cols] = data
        # diagonal d holds data[c][(c + d) mod padded] for every database row c
        c = np.arange(rows)
        diagonals = np.stack([wide[c, (c + d) % padded] for d in range(padded)])
        per_column = -(-rows // n)
        full = np.zeros((padded, per_column * n), dtype=np.uint64)
        full[:, :rows] = diagonals
        chunks = full.reshape(padded, per_column, n)
        half = n // 2
        for d in range(padded):
            step = d // bsgs.babyStep * bsgs.babyStep
            if step:
                chunks[d] = np.concatenate([np.roll(chunks[d][:, :half], step, axis=1),
                                            np.roll(chunks[d][:, half:], step, axis=1)], axis=1)
        return SimdEncoder(n, t).encode(chunks.reshape(padded * per_column, n))

    def mulTranspose(self, vector, evaluationKey: EvaluationKey, modSwitchDownToSingle: bool = False) -> np.ndarray:
        """mulTranspose(vector:using:) for one (2, L, N) or a batch (batch, 2, L, N) of dense-row query ciphertexts.
        Returns (batch, resultCiphertextCount, 2, L or 1, N)."""
        ctx = self.context
        cts = _host(vector)
        words = 2 * ctx.L * ctx.degree
        if cts.size % words:
            raise HeError(-1, "invalidCiphertext: query vectors must be ciphertexts of 2 x L x N")
        batch = cts.size // words
        out = np.empty((batch, self.resultCiphertextCount, 2, 1 if modSwitchDownToSingle else ctx.L, ctx.degree), dtype=np.uint64)
        _check(load_library().hecuda_pnns_mul_transpose_vector(ctx._h, evaluationKey._h, self._h, _ptr(cts), batch,
                                                              1 if modSwitchDownToSingle else 0, _ptr(out)))
        return out

    def mulTransposeMatrix(self, ciphertexts, queryDimensions: MatrixDimensions, evaluationKey: EvaluationKey,
                           modSwitchDownToSingle: bool = False) -> np.ndarray:
        """mulTranspose(matrix:using:) (MatrixMultiplication.swift:236-298): `ciphertexts` is the dense-row packed query
        CiphertextMatrix (count, 2, L, N); returns the dense-column packed result ciphertexts (count', 2, L or 1, N)."""
        ctx = self.context
        n = ctx.degree
        cts = _host(ciphertexts)
        words = 2 * ctx.L * n
        count = cts.size // words
        self._checkQuery(queryDimensions, count, cts.size % words == 0)
        d = self._rowDescriptors(queryDimensions, count, evaluationKey.galoisElements)
        out = np.empty((d["capacity"], 2, 1 if modSwitchDownToSingle else ctx.L, n), dtype=np.uint64)
        produced = C.c_int64(0)
        _check(load_library().hecuda_pnns_mul_transpose_matrix(
            ctx._h, evaluationKey._h, self._h, _ptr(cts), count, queryDimensions.rowCount, d["index"], _ptr(d["masks"]),
            d["rotate"], d["step"], d["plan"], d["planCount"], 1 if modSwitchDownToSingle else 0, _ptr(out), d["capacity"],
            C.byref(produced)))
        return out[: produced.value]

    def computeResponses(self, ciphertexts, queryDimensions: MatrixDimensions, evaluationKeys) -> np.ndarray:
        """Server.computeResponse (Server.swift:61-88) for many clients in one C-ABI call
        (hecuda_pnns_compute_response_clients): client c's dense-row query ciphertexts with evaluationKeys[c], its replies
        bit-identical to `mulTransposeMatrix(ciphertexts[c], queryDimensions, evaluationKeys[c], modSwitchDownToSingle=True)`.
        Groups of up to HECUDA_PNNS_CLIENT_GROUP clients share every pass, including one pass over the matrix.  The
        packing rotations are planned with the first key's Galois elements (every key must hold them).

        ciphertexts: (clients, count, 2, L, N) Coeff.  Returns (clients, count', 2, 1, N)."""
        ctx = self.context
        n = ctx.degree
        keys = list(evaluationKeys)
        cts = _host(ciphertexts)
        words = 2 * ctx.L * n
        if not keys or cts.size % (words * len(keys)):
            raise HeError(-1, "invalidCiphertext: ciphertexts must be one query of 2 x L x N ciphertexts per evaluation key")
        count = cts.size // (words * len(keys))
        self._checkQuery(queryDimensions, count, True)
        d = self._rowDescriptors(queryDimensions, count, keys[0].galoisElements)
        out = np.empty((len(keys), d["capacity"], 2, 1, n), dtype=np.uint64)
        produced = C.c_int64(0)
        key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
        _check(load_library().hecuda_pnns_compute_response_clients(
            ctx._h, key_handles, len(keys), self._h, _ptr(cts), count, queryDimensions.rowCount, d["index"], _ptr(d["masks"]),
            d["rotate"], d["step"], d["plan"], d["planCount"], _ptr(out), d["capacity"], C.byref(produced)))
        return out[:, : produced.value]

    def _checkQuery(self, queryDimensions: MatrixDimensions, count: int, whole: bool):
        if queryDimensions.columnCount != self.dimensions.columnCount:
            raise PnnsError(f"invalidMatrixDimensions(rowCount: {queryDimensions.rowCount}, columnCount: {queryDimensions.columnCount})")
        expected = CiphertextMatrix.ciphertextCount(self.context.degree, queryDimensions)
        if not whole or count != expected:
            raise PnnsError(f"wrongCiphertextCount(got: {count}, expected: {expected})")

    def _rowDescriptors(self, queryDimensions: MatrixDimensions, count: int, galoisElements) -> dict:
        """What extractDenseRow derives for every query row, and the packing rotations, as the C ABI takes them."""
        n = self.context.degree
        rows = queryDimensions.rowCount
        index = (C.c_int32 * rows)()
        rotate = (C.c_int32 * rows)()
        masks = np.zeros((rows, n), dtype=np.uint64)
        if rows > 1:
            encoder = SimdEncoder(n, self.context.plaintextModulus)
            values = np.zeros((rows, n), dtype=np.uint64)
            for r in range(rows):
                index[r], mask, rotate[r] = CiphertextMatrix.denseRowExtraction(n, queryDimensions, count, r)
                values[r, : len(mask)] = mask
            masks = encoder.encode(values)
        per_simd_row = (n // 2) // self.dimensions.rowCount
        sequence = []
        if per_simd_row > 1 and rows > 1:
            sequence = GaloisElement.rotationSequence(galoisElements, self.dimensions.rowCount, n)
        return dict(index=index, rotate=rotate, masks=masks, step=_next_power_of_two(queryDimensions.columnCount),
                    plan=(C.c_int32 * max(1, len(sequence)))(*sequence), planCount=len(sequence),
                    capacity=rows * self.resultCiphertextCount)

    def close(self):
        if getattr(self, "_h", None) is not None:
            load_library().hecuda_pnns_matrix_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PnnsWire:
    """Request / reply bytes of the PNNS server (the payloads of the reference's protobuf messages)."""

    @staticmethod
    def computeResponses(matrix: PlaintextMatrix, queryPoly0, querySeeds, queryDimensions: MatrixDimensions, evaluationKeys):
        """PlaintextMatrix.computeResponses on the wire, one C-ABI call (hecuda_pnns_compute_response_clients_wire): the
        queries as seeded serialized ciphertexts (SerializedCiphertext.seeded), the replies serialized forDecryption
        (PnnsConversionApi.swift:48) with skipLSBsForDecryption.
        queryPoly0: (clients, count, byteCount(L rows)) uint8; querySeeds: (clients, count, 32) uint8.  Returns
        (replies, skipLSBs) with replies of shape (clients, count', bytes(poly0) + bytes(poly1))."""
        from . import Bfv
        from .pir import skipLSBsForDecryption
        ctx = matrix.context
        keys = list(evaluationKeys)
        seeds = np.ascontiguousarray(np.asarray(querySeeds, dtype=np.uint8))
        poly0 = np.ascontiguousarray(np.asarray(queryPoly0, dtype=np.uint8))
        size = Bfv.serializationByteCount(ctx, ctx.L)
        if not keys or seeds.size % (32 * len(keys)):
            raise HeError(-1, "serializedBufferSizeMismatch: querySeeds must be one set of 32-byte seeds per evaluation key")
        count = seeds.size // (32 * len(keys))
        if poly0.size != len(keys) * count * size:
            raise HeError(-1, f"serializedBufferSizeMismatch(poly0: {poly0.size} bytes, expected {len(keys) * count * size})")
        matrix._checkQuery(queryDimensions, count, True)
        d = matrix._rowDescriptors(queryDimensions, count, keys[0].galoisElements)
        skips = skipLSBsForDecryption(ctx)
        sizes = [Bfv.serializationByteCount(ctx, 1, s) for s in skips]
        out = np.empty((len(keys), d["capacity"], sum(sizes)), dtype=np.uint8)
        produced = C.c_int64(0)
        key_handles = (C.c_void_p * len(keys))(*[k._h for k in keys])
        _check(load_library().hecuda_pnns_compute_response_clients_wire(
            ctx._h, key_handles, len(keys), matrix._h, poly0.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p),
            count, queryDimensions.rowCount, d["index"], _ptr(d["masks"]), d["rotate"], d["step"], d["plan"], d["planCount"],
            skips[0], skips[1], out.ctypes.data_as(C.c_void_p), d["capacity"], C.byref(produced)))
        return out[:, : produced.value], skips


class PnnsRequestFields(C.Structure):
    """hecuda_pnns_request_fields (include/hecuda.h)."""
    _fields_ = [("query_count", C.c_int32), ("query_row_count", C.c_uint32), ("has_evaluation_key", C.c_int32),
                ("has_key_metadata", C.c_int32), ("shard_index_count", C.c_int64), ("shard_id_count", C.c_int64),
                ("config_id_offset", C.c_uint64), ("config_id_bytes", C.c_uint64),
                ("evaluation_key_offset", C.c_uint64), ("evaluation_key_bytes", C.c_uint64),
                ("key_timestamp", C.c_uint64), ("key_identifier_offset", C.c_uint64), ("key_identifier_bytes", C.c_uint64)]


class PnnsShardResponseShape(C.Structure):
    """hecuda_pnns_shard_response_shape (include/hecuda.h)."""
    _fields_ = [("matrix_count", C.c_int32), ("reply_count", C.c_int32), ("row_count", C.c_uint32),
                ("column_count", C.c_uint32), ("id_count", C.c_int64), ("metadata_count", C.c_int64)]


class PnnsRequest:
    """api.pnns.v1.PNNSRequest, the envelope a PNNS server receives."""

    @staticmethod
    def fields(message) -> dict:
        """The walk of a PNNSRequest (hecuda_pnns_request_fields_read), nothing copied on the host side: queryCount and
        queryRowCount (the matrices' common num_rows), configId, the key metadata (keyTimestamp, keyIdentifier; from
        evaluation_key_metadata, or evaluation_key.metadata when that is absent), the (offset, length) range of
        evaluation_key.evaluation_key (a SerializedEvaluationKey for EvaluationKey.fromProtoMany; None when unset),
        shardIndices and shardIds.  Routing by shard and caching keys by identifier stay the caller's."""
        b = bytes(message)
        r = PnnsRequestFields()
        lib = load_library()
        _check(lib.hecuda_pnns_request_fields_read(b, len(b), C.byref(r), None, 0, None, 0))
        indices = (C.c_uint32 * max(1, r.shard_index_count))()
        ranges = (C.c_uint64 * max(2, 2 * r.shard_id_count))()
        _check(lib.hecuda_pnns_request_fields_read(b, len(b), C.byref(r), indices, r.shard_index_count, ranges,
                                                   r.shard_id_count))

        def span(offset, size):
            return b[offset:offset + size]

        return {
            "queryCount": r.query_count,
            "queryRowCount": r.query_row_count,
            "configId": span(r.config_id_offset, r.config_id_bytes),
            "keyTimestamp": r.key_timestamp if r.has_key_metadata else None,
            "keyIdentifier": span(r.key_identifier_offset, r.key_identifier_bytes) if r.has_key_metadata else None,
            "evaluationKey": (r.evaluation_key_offset, r.evaluation_key_bytes) if r.has_evaluation_key else None,
            "shardIndices": list(indices[:r.shard_index_count]),
            "shardIds": [span(ranges[2 * i], ranges[2 * i + 1]).decode() for i in range(r.shard_id_count)],
        }


def _message_buffers(messages):
    buffers = [np.frombuffer(m, dtype=np.uint8) if isinstance(m, (bytes, bytearray, memoryview)) else
               np.ascontiguousarray(m, dtype=np.uint8).reshape(-1) for m in messages]
    keep = [b if b.size else np.zeros(1, np.uint8) for b in buffers]
    counts = np.array([b.size for b in buffers], dtype=np.uint64)
    return (C.c_void_p * len(keep))(*[b.ctypes.data for b in keep]), counts, keep


def denseRowVector(context, vector) -> np.ndarray:
    """The SIMD values of a one-row `.denseRow` matrix (PlaintextMatrix.swift:341-413): the row padded to a power of
    two and repeated to fill both SIMD rows.  Returns the coefficient plaintext (N,)."""
    n, t = context.degree, context.plaintextModulus
    v = [int(x) % t for x in vector]
    packed = v + [0] * (_next_power_of_two(len(v)) - len(v))
    columns = n // 2
    if len(packed) < columns < len(packed) + len(v):
        packed += [0] * (columns - len(packed))
    offset = len(packed) % columns
    if offset:
        packed += [0] * (_next_power_of_two(offset) - offset)
    repeat = list(packed) if len(packed) <= columns else packed[columns:]
    while len(packed) < n:
        packed += repeat
    return SimdEncoder(n, t).encode(np.array(packed[:n], dtype=np.uint64))[0]


# ------------------------------------------------------------------------------------------------ client and server
# Client, Server, Database and ProcessedDatabase of PrivateNearestNeighborSearch (Client.swift, Server.swift,
# Database.swift, ProcessedDatabase.swift, Config.swift) over one context per plaintext modulus.  Float vectors are
# normalised, scaled and rounded on the device in Swift Float arithmetic; queries are packed, encoded and encrypted
# there (hecuda_pnns_query_generate), and replies decrypted, decoded, CRT-composed and turned into float distances
# (hecuda_pnns_decrypt_distances).

COSINE_SIMILARITY = "cosineSimilarity"  # DistanceMetric.cosineSimilarity, the only metric


@dataclass(frozen=True)
class EncryptionParameters:
    """The parts of EncryptionParameters a PNNS configuration compares contexts against."""

    polyDegree: int
    plaintextModulus: int
    coefficientModuli: tuple

    @staticmethod
    def ofContext(context: Context) -> "EncryptionParameters":
        return EncryptionParameters(context.degree, context.plaintextModulus, tuple(context.coefficientModuli))


class MatrixMultiplication:
    @staticmethod
    def evaluationKeyConfig(plaintextMatrixDimensions: MatrixDimensions, maxQueryCount: int, degree: int):
        """MatrixMultiplication.evaluationKeyConfig (MatrixMultiplication.swift:76-116) united with
        CiphertextMatrix.extractDenseRowConfig (CiphertextMatrix.swift:224-243)."""
        from .pir import EvaluationKeyConfig
        simd_columns = degree // 2
        bsgs = BabyStepGiantStep.forVectorDimension(plaintextMatrixDimensions.columnCount)
        rot = GaloisElement.rotatingColumns
        elements = [rot(-1, degree), rot(-bsgs.babyStep, degree), GaloisElement.swappingRows(degree)]
        if simd_columns // plaintextMatrixDimensions.rowCount > 1:
            elements.append(rot(1, degree))
            if simd_columns > 16:
                elements.append(rot(16, degree))
            if simd_columns > 256:
                elements.append(rot(256, degree))
        if maxQueryCount != 1:
            width = _next_power_of_two(plaintextMatrixDimensions.columnCount)
            if width != simd_columns:
                elements.append(rot(width, degree))
        return EvaluationKeyConfig(list(dict.fromkeys(elements)), False)


class ClientConfig:
    """ClientConfig (Config.swift:50-136).  encryptionParameters: the first context's EncryptionParameters; one more
    set per extra plaintext modulus, identical but for t."""

    def __init__(self, encryptionParameters: EncryptionParameters, scalingFactor: int, vectorDimension: int,
                 evaluationKeyConfig, distanceMetric: str = COSINE_SIMILARITY, extraPlaintextModuli=(),
                 queryPacking="denseRow", errorStdDev: float = 3.2, securityLevel: str = "unchecked"):
        """queryPacking: "denseRow", "denseColumn" or a BabyStepGiantStep (.diagonal).  errorStdDev: 3.2 (.stdDev32) or
        6.4 (.stdDev64); securityLevel: "unchecked" or "quantum128", which EncryptionParameters.init checks
        (EncryptionParameters.swift:139-145): insecureEncryptionParameters when log2 of the coefficient modulus exceeds
        the bound for the degree."""
        p = encryptionParameters
        self.encryptionParameters = [p] + [EncryptionParameters(p.polyDegree, int(t), p.coefficientModuli)
                                           for t in extraPlaintextModuli]
        self.scalingFactor = int(scalingFactor)
        self.queryPacking = queryPacking
        self.vectorDimension = int(vectorDimension)
        self.evaluationKeyConfig = evaluationKeyConfig
        self.distanceMetric = distanceMetric
        self.extraPlaintextModuli = [int(t) for t in extraPlaintextModuli]
        self.errorStdDev, self.securityLevel = float(errorStdDev), securityLevel
        _check_security(p, self.errorStdDev, securityLevel)

    def serialize(self) -> bytes:
        """The ClientConfig protobuf message (PnnsConversion.swift: ClientConfig.proto()), as SwiftProtobuf writes it."""
        return _serialize_config(load_library().hecuda_pnns_client_config_serialize, _config_struct(self))

    @staticmethod
    def deserialize(data) -> "ClientConfig":
        """ClientConfig.native() of a ClientConfig protobuf message, with the reference's refusals."""
        return _client_config(_parse_config(load_library().hecuda_pnns_client_config_parse, data))

    @property
    def plaintextModuli(self):
        return [p.plaintextModulus for p in self.encryptionParameters]

    @staticmethod
    def maxScalingFactor(distanceMetric: str, vectorDimension: int, plaintextModuli) -> int:
        """ClientConfig.maxScalingFactor (Config.swift:112-120) in Float: floor(sqrt((t - 1) / 2) - sqrt(d) / 2) with
        t the Float product of the moduli."""
        if distanceMetric != COSINE_SIMILARITY:
            raise PnnsError(f"wrongDistanceMetric(got: {distanceMetric}, expected: {COSINE_SIMILARITY})")
        f = np.float32
        t = f(1)
        for m in plaintextModuli:
            t = f(t * f(int(m)))
        value = f(np.sqrt(f(f(t - f(1)) / f(2)))) - f(f(np.sqrt(f(int(vectorDimension)))) / f(2))
        return int(np.floor(f(value)))

    def validateContexts(self, contexts):
        """ClientConfig.validateContexts (Config.swift:125-135)."""
        if len(contexts) != len(self.encryptionParameters):
            raise PnnsError(f"wrongContextsCount(got: {len(contexts)}, expected: {len(self.encryptionParameters)})")
        for context, params in zip(contexts, self.encryptionParameters):
            got = EncryptionParameters.ofContext(context)
            if got != params:
                raise PnnsError(f"wrongEncryptionParameters(got: {got}, expected: {params})")


class ServerConfig:
    """ServerConfig (Config.swift:138-204): the client's configuration and the database's .diagonal packing."""

    def __init__(self, clientConfig: ClientConfig, babyStepGiantStep: BabyStepGiantStep = None):
        self.clientConfig = clientConfig
        self.babyStepGiantStep = babyStepGiantStep or BabyStepGiantStep.forVectorDimension(clientConfig.vectorDimension)

    def __getattr__(self, name):  # scalingFactor, plaintextModuli, distanceMetric, vectorDimension, ...
        if name == "clientConfig":
            raise AttributeError(name)
        return getattr(self.clientConfig, name)

    def validateContexts(self, contexts):
        self.clientConfig.validateContexts(contexts)

    def serialize(self) -> bytes:
        """The ServerConfig protobuf message (PnnsConversion.swift: ServerConfig.proto()), as SwiftProtobuf writes it."""
        return _serialize_config(load_library().hecuda_pnns_server_config_serialize,
                                 _config_struct(self.clientConfig, self.babyStepGiantStep))

    @staticmethod
    def deserialize(data) -> "ServerConfig":
        """ServerConfig.native() of a ServerConfig protobuf message.  Its database packing must be .diagonal, the only
        one resident here (HeError, unsupported, otherwise)."""
        return _server_config(_parse_config(load_library().hecuda_pnns_server_config_parse, data))


# ---- the configuration messages: hecuda_pnns_server_config, filled and read here; the protobuf bytes are the library's
_MAX_MODULI, _MAX_EXTRA, _MAX_GALOIS = 32, 7, 64  # HECUDA_PNNS_MAX_*
_PACKINGS = {"denseRow": 1, "diagonal": 2, "denseColumn": 3}
_ERR_UNSUPPORTED = -2  # HECUDA_ERR_UNSUPPORTED


class _ConfigStruct(C.Structure):  # hecuda_pnns_server_config
    _fields_ = [("poly_degree", C.c_uint64), ("plaintext_modulus", C.c_uint64), ("coefficient_moduli_count", C.c_int32),
                ("error_std_dev", C.c_int32), ("coefficient_moduli", C.c_uint64 * _MAX_MODULI),
                ("security_level", C.c_int32), ("he_scheme", C.c_int32), ("scaling_factor", C.c_uint64),
                ("query_packing", C.c_int32), ("query_vector_dimension", C.c_uint32), ("query_baby_step", C.c_uint32),
                ("query_giant_step", C.c_uint32), ("vector_dimension", C.c_uint32), ("galois_element_count", C.c_int32),
                ("galois_elements", C.c_uint32 * _MAX_GALOIS), ("distance_metric", C.c_int32),
                ("extra_plaintext_moduli_count", C.c_int32), ("extra_plaintext_moduli", C.c_uint64 * _MAX_EXTRA),
                ("database_packing", C.c_int32), ("database_vector_dimension", C.c_uint32),
                ("database_baby_step", C.c_uint32), ("database_giant_step", C.c_uint32)]


def _check_security(params: EncryptionParameters, errorStdDev: float, securityLevel: str):
    from . import _MAX_LOG2_Q_STDDEV32, _MAX_LOG2_Q_STDDEV64
    if errorStdDev not in (3.2, 6.4):
        raise PnnsError(f"invalidEncryptionParameters: errorStdDev must be 3.2 (.stdDev32) or 6.4 (.stdDev64), got {errorStdDev}")
    if securityLevel == "unchecked":
        return
    if securityLevel != "quantum128":
        raise PnnsError(f"invalidEncryptionParameters: securityLevel must be 'unchecked' or 'quantum128', got {securityLevel!r}")
    table = _MAX_LOG2_Q_STDDEV64 if errorStdDev == 6.4 else _MAX_LOG2_Q_STDDEV32
    if params.polyDegree not in table:
        raise PnnsError(f"invalidEncryptionParameters: no quantum128 bound for degree {params.polyDegree}, "
                        f"errorStdDev {errorStdDev}")
    log2q = np.float32(0)
    for q in params.coefficientModuli:  # Float arithmetic, as the reference sums it
        log2q = np.float32(log2q + np.log2(np.float32(q)))
    if log2q > np.float32(table[params.polyDegree]):
        raise PnnsError(f"insecureEncryptionParameters: log2(q) = {float(log2q):.2f} exceeds {table[params.polyDegree]} "
                        f"for degree {params.polyDegree}")


def _set_packing(s, prefix: str, packing):
    if isinstance(packing, BabyStepGiantStep):
        setattr(s, prefix + "_packing", 2)
        setattr(s, prefix + "_vector_dimension", packing.vectorDimension)
        setattr(s, prefix + "_baby_step", packing.babyStep)
        setattr(s, prefix + "_giant_step", packing.giantStep)
    elif packing in ("denseRow", "denseColumn"):
        setattr(s, prefix + "_packing", _PACKINGS[packing])
    else:
        raise PnnsError(f"unknown packing {packing!r}")


def _packing(s, prefix: str):
    kind = getattr(s, prefix + "_packing")
    if kind == 2:
        return BabyStepGiantStep(getattr(s, prefix + "_vector_dimension"), getattr(s, prefix + "_baby_step"),
                                 getattr(s, prefix + "_giant_step"))
    return {1: "denseRow", 3: "denseColumn"}[kind]


def _config_struct(config: ClientConfig, databasePacking: BabyStepGiantStep = None) -> _ConfigStruct:
    _check_metric(config.distanceMetric)
    _check_security(config.encryptionParameters[0], config.errorStdDev, config.securityLevel)
    p = config.encryptionParameters[0]
    galois = list(config.evaluationKeyConfig.galoisElements)
    if len(p.coefficientModuli) > _MAX_MODULI or len(config.extraPlaintextModuli) > _MAX_EXTRA or len(galois) > _MAX_GALOIS:
        raise HeError(_ERR_UNSUPPORTED, "a configuration with more moduli or Galois elements than hecuda_pnns_server_config holds")
    s = _ConfigStruct()
    s.poly_degree, s.plaintext_modulus = p.polyDegree, p.plaintextModulus
    s.coefficient_moduli_count = len(p.coefficientModuli)
    s.coefficient_moduli[:len(p.coefficientModuli)] = [int(q) for q in p.coefficientModuli]
    s.error_std_dev = 1 if config.errorStdDev == 6.4 else 0
    s.security_level = 1 if config.securityLevel == "quantum128" else 0
    s.he_scheme = 1  # BFV
    s.scaling_factor = config.scalingFactor
    _set_packing(s, "query", config.queryPacking)
    s.vector_dimension = config.vectorDimension
    s.galois_element_count = len(galois)
    s.galois_elements[:len(galois)] = [int(g) for g in galois]
    s.distance_metric = 0  # cosineSimilarity
    s.extra_plaintext_moduli_count = len(config.extraPlaintextModuli)
    s.extra_plaintext_moduli[:len(config.extraPlaintextModuli)] = config.extraPlaintextModuli
    if databasePacking is not None:
        _set_packing(s, "database", databasePacking)
    return s


def _client_config(s: _ConfigStruct) -> ClientConfig:
    from .pir import EvaluationKeyConfig
    params = EncryptionParameters(int(s.poly_degree), int(s.plaintext_modulus),
                                  tuple(int(q) for q in s.coefficient_moduli[:s.coefficient_moduli_count]))
    return ClientConfig(params, int(s.scaling_factor), int(s.vector_dimension),
                        EvaluationKeyConfig([int(g) for g in s.galois_elements[:s.galois_element_count]], False),
                        COSINE_SIMILARITY, [int(t) for t in s.extra_plaintext_moduli[:s.extra_plaintext_moduli_count]],
                        _packing(s, "query"), 6.4 if s.error_std_dev == 1 else 3.2,
                        "quantum128" if s.security_level == 1 else "unchecked")


def _server_config(s: _ConfigStruct) -> ServerConfig:
    packing = _packing(s, "database")
    if not isinstance(packing, BabyStepGiantStep):
        raise HeError(_ERR_UNSUPPORTED, f"databasePacking .{packing}: only .diagonal matrices are resident here")
    return ServerConfig(_client_config(s), packing)


def _parse_config(parse, data) -> _ConfigStruct:
    buf = np.frombuffer(bytes(data) or b"\0", dtype=np.uint8)
    s = _ConfigStruct()
    _check(parse(_ptr(buf), len(bytes(data)), C.byref(s)))
    return s


def _serialize_config(serialize, s: _ConfigStruct) -> bytes:
    size = C.c_uint64(0)
    _check(serialize(C.byref(s), None, 0, C.byref(size)))
    out = np.empty(max(1, size.value), dtype=np.uint8)
    _check(serialize(C.byref(s), _ptr(out), out.size, C.byref(size)))
    return out[:size.value].tobytes()


def _check_metric(metric: str):
    if metric != COSINE_SIMILARITY:
        raise PnnsError(f"wrongDistanceMetric(got: {metric}, expected: {COSINE_SIMILARITY})")


def _float_rows(vectors) -> np.ndarray:
    v = np.ascontiguousarray(np.asarray(vectors, dtype=np.float32))
    return v.reshape(1, -1) if v.ndim == 1 else v


@dataclass
class DatabaseRow:
    """DatabaseRow (Database.swift): an identifier, optional metadata bytes and the vector."""

    entryId: int
    entryMetadata: bytes
    vector: list


@dataclass
class Database:
    rows: list


@dataclass
class Query:
    """Query (PnnsProtocol.swift:18-27): one dense-row ciphertext matrix per plaintext modulus, each (count, 2, L, N)
    Coeff, or with `wire` each the .seeded form (poly0 (count, B) uint8, seeds (count, 32) uint8)."""

    ciphertextMatrices: list
    dimensions: MatrixDimensions
    wire: bool = False


@dataclass
class Response:
    """Response (PnnsProtocol.swift:30-52): one dense-column ciphertext matrix per plaintext modulus of `dimensions`
    (database rows x query rows), each (count, 2, l, N) Coeff or PnnsWire reply bytes (bytes (count, B0 + B1), skips)."""

    ciphertextMatrices: list
    dimensions: MatrixDimensions
    entryIds: list = None
    entryMetadatas: list = None

    def _ciphertexts(self, contexts):
        from . import Bfv
        out = []
        for ctx, m in zip(contexts, self.ciphertextMatrices):
            if isinstance(m, tuple):  # PnnsWire reply bytes, skipLSBsForDecryption
                data, skips = m
                data = np.asarray(data, dtype=np.uint8).reshape(-1, np.asarray(data).shape[-1])
                b0 = Bfv.serializationByteCount(ctx, 1, skips[0])
                poly0 = Bfv.load(ctx, np.ascontiguousarray(data[:, :b0]), 1, skips[0])
                poly1 = Bfv.load(ctx, np.ascontiguousarray(data[:, b0:]), 1, skips[1])
                m = np.stack([poly0, poly1], axis=1)
            out.append(np.ascontiguousarray(np.asarray(m, dtype=np.uint64)))
        return out

    def noiseBudget(self, contexts, secretKey) -> float:
        """Response.noiseBudget (PnnsProtocol.swift:98-102): the least budget over the matrices, each under its own
        context's t.  Must never be forwarded to another party."""
        from . import Bfv
        budgets = [float(np.min(Bfv.noiseBudget(ctx, secretKey, cts)))
                   for ctx, cts in zip(contexts, self._ciphertexts(contexts))]
        return min(budgets) if budgets else -math.inf


@dataclass
class DatabaseDistances:
    """DatabaseDistances (PnnsProtocol.swift:55-77): float32 distances (database rows x query rows)."""

    distances: np.ndarray
    entryIds: list
    entryMetadatas: list


class Client:
    """Client (Client.swift:20-147) over one context per plaintext modulus."""

    def __init__(self, config: ClientConfig, contexts):
        _check_metric(config.distanceMetric)
        if config.errorStdDev != 3.2:
            raise HeError(_ERR_UNSUPPORTED, f"errorStdDev {config.errorStdDev}: the device samples errors at 3.2 only")
        config.validateContexts(contexts)
        ts = config.plaintextModuli
        if len(set(ts)) != len(ts):
            raise PnnsError("plaintext moduli must be pairwise distinct")
        self.config, self.contexts = config, list(contexts)

    @property
    def evaluationKeyConfig(self):
        return self.config.evaluationKeyConfig

    def generateSecretKey(self, seed=None):
        from . import SecretKey
        return SecretKey.generate(self.contexts[0], seed)

    def generateEvaluationKey(self, secretKey):
        """On contexts[0], used with every plaintext modulus (Client.swift:137-146)."""
        return EvaluationKey.generate(self.contexts[0], self.evaluationKeyConfig, secretKey)

    def generateQuery(self, vectors, secretKey, wire: bool = False, aSeeds=None, errorSeeds=None) -> Query:
        """Client.generateQuery (Client.swift:73-91) on the device: one encrypted .denseRow matrix per context, the values
        reduced mod t when there are several (hecuda_pnns_query_generate).  Seeds: per context, (count, 32) uint8 each,
        fresh from secrets.token_bytes by default."""
        from . import Bfv, _secret_poly, _seeds
        v = _float_rows(vectors)
        rows, cols = v.shape
        dims = MatrixDimensions(rows, cols)
        sk = _secret_poly(secretKey)
        reduce = 1 if len(self.contexts) > 1 else 0
        out = []
        for k, ctx in enumerate(self.contexts):
            count = CiphertextMatrix.ciphertextCount(ctx.degree, dims) if cols <= ctx.degree // 2 else 1
            a = _seeds(count, None if aSeeds is None else aSeeds[k])
            err = _seeds(count, None if errorSeeds is None else errorSeeds[k])
            if wire:
                poly0 = np.empty((count, Bfv.serializationByteCount(ctx, ctx.L)), dtype=np.uint8)
                cts = None
            else:
                cts = np.empty((count, 2, ctx.L, ctx.degree), dtype=np.uint64)
                poly0 = None
            rc = load_library().hecuda_pnns_query_generate(
                ctx._h, _ptr(sk), v.ctypes.data_as(C.c_void_p), rows, cols, self.config.scalingFactor, reduce, _ptr(a),
                _ptr(err), _ptr(cts) if cts is not None else None, _ptr(poly0) if poly0 is not None else None)
            err[:] = 0
            _check(rc)
            out.append((poly0, a) if wire else cts)
        return Query(out, dims, wire)

    def evaluationKeyMessage(self, secretKey):
        """generateEvaluationKey as the reference's client sends it: (key, SerializedEvaluationKey.proto() bytes) of a
        seeded key on contexts[0]."""
        from .pir import evaluationKeyMessage
        key, form = EvaluationKey.generate(self.contexts[0], self.evaluationKeyConfig, secretKey, wire=True)
        return key, evaluationKeyMessage(self.contexts[0], form)

    def requestMessage(self, vectors, secretKey, evaluationKey=None, keyTimestamp: int = 0, keyIdentifier: bytes = b"",
                       configId: bytes = b"", aSeeds=None, errorSeeds=None) -> bytes:
        """generateQuery as the reference's client sends it: Query.proto() in an api.pnns.v1.PNNSRequest
        (hecuda_pnns_request_write), one .denseRow matrix of .seeded ciphertexts per plaintext modulus, with
        generateQuery(wire=True)'s seeds.  evaluationKey: a SerializedEvaluationKey message (evaluationKeyMessage's
        bytes) to send in evaluation_key, with its metadata; configId: the PNNSConfig identifier."""
        query = self.generateQuery(vectors, secretKey, wire=True, aSeeds=aSeeds, errorSeeds=errorSeeds)
        from .pir import _written
        poly0 = [np.ascontiguousarray(m[0]) for m in query.ciphertextMatrices]
        seeds = [np.ascontiguousarray(m[1]) for m in query.ciphertextMatrices]
        count = seeds[0].shape[0]
        K = len(self.contexts)
        ctxs = (C.c_void_p * K)(*[c._h.value for c in self.contexts])
        p0 = (C.c_void_p * K)(*[a.ctypes.data for a in poly0])
        sd = (C.c_void_p * K)(*[a.ctypes.data for a in seeds])
        key = bytes(evaluationKey) if evaluationKey is not None else None
        ident, config = bytes(keyIdentifier), bytes(configId)
        return _written(lambda out, capacity, written: load_library().hecuda_pnns_request_write(
            ctxs, K, query.dimensions.rowCount, query.dimensions.columnCount, p0, sd, count, config or None, len(config),
            key, len(key) if key is not None else 0, keyTimestamp, ident or None, len(ident), out, capacity, written))

    def decryptResponseMessage(self, message, secretKey) -> DatabaseDistances:
        """decrypt of an api.pnns.v1.PNNSShardResponse: its matrices found by hecuda_pnns_shard_response_read, each
        reply's polys loaded with its matrix's skip bits, then decrypt; the entry ids and metadata from the message."""
        b = np.frombuffer(bytes(message), dtype=np.uint8)
        buf = b if b.size else np.zeros(1, np.uint8)
        K = len(self.contexts)
        ctxs = (C.c_void_p * K)(*[c._h.value for c in self.contexts])
        lib = load_library()
        shape = PnnsShardResponseShape()
        _check(lib.hecuda_pnns_shard_response_read(ctxs, K, buf.ctypes.data_as(C.c_void_p), b.size, C.byref(shape), None,
                                                   None, None, None))
        offsets = np.empty(max(1, K * shape.reply_count), dtype=np.uint64)
        skips = np.empty(2 * K, dtype=np.int32)
        ids = np.empty(max(1, shape.id_count), dtype=np.uint64)
        ranges = np.empty(max(2, 2 * shape.metadata_count), dtype=np.uint64)
        _check(lib.hecuda_pnns_shard_response_read(ctxs, K, buf.ctypes.data_as(C.c_void_p), b.size, C.byref(shape),
                                                   _ptr(offsets), skips.ctypes.data_as(C.c_void_p), _ptr(ids), _ptr(ranges)))
        from . import Bfv
        matrices = []
        for k, ctx in enumerate(self.contexts):
            s = [int(skips[2 * k]), int(skips[2 * k + 1])]
            size = sum(Bfv.serializationByteCount(ctx, 1, x) for x in s)
            rows = np.stack([b[int(o):int(o) + size] for o in offsets[k * shape.reply_count:(k + 1) * shape.reply_count]])
            matrices.append((rows, s))
        metadata = [b[int(ranges[2 * i]):int(ranges[2 * i] + ranges[2 * i + 1])].tobytes()
                    for i in range(shape.metadata_count)]
        response = Response(matrices, MatrixDimensions(shape.row_count, shape.column_count),
                            [int(v) for v in ids[:shape.id_count]], metadata)
        return self.decrypt(response, secretKey)

    def decrypt(self, response: Response, secretKey) -> DatabaseDistances:
        """Client.decrypt (Client.swift:99-127) on the device (hecuda_pnns_decrypt_distances): float32 distances,
        database rows x query rows."""
        from . import _secret_poly
        if not response.ciphertextMatrices:
            raise PnnsError("emptyCiphertextArray")
        if len(response.ciphertextMatrices) != len(self.contexts):
            raise PnnsError(f"wrongCiphertextMatrixCount(got: {len(response.ciphertextMatrices)}, expected: {len(self.contexts)})")
        cts = response._ciphertexts(self.contexts)
        count, polys, l, n = cts[0].shape
        if polys != 2 or any(c.shape != cts[0].shape for c in cts):
            raise HeError(-1, "invalidCiphertext: every matrix must hold the same number of 2 x l x N ciphertexts")
        sk = _secret_poly(secretKey)
        dims = response.dimensions
        out = np.empty((dims.rowCount, dims.columnCount), dtype=np.float32)
        ctxs = (C.c_void_p * len(self.contexts))(*[c._h.value for c in self.contexts])
        replies = (C.c_void_p * len(cts))(*[c.ctypes.data for c in cts])
        _check(load_library().hecuda_pnns_decrypt_distances(ctxs, len(self.contexts), _ptr(sk), replies, count, l,
                                                           dims.rowCount, dims.columnCount, self.config.scalingFactor,
                                                           out.ctypes.data_as(C.c_void_p)))
        return DatabaseDistances(out, response.entryIds, response.entryMetadatas)


@dataclass
class ValidationResult:
    """ValidationResult (ProcessedDatabase.swift:147-184): the first trial's key and query, the last response, its
    distances (first trial), the least noise budget and each trial's response time in seconds."""

    evaluationKey: Any
    query: Query
    response: Response
    databaseDistances: DatabaseDistances
    noiseBudget: float
    computeTimes: list


class ProcessedDatabase:
    """ProcessedDatabase (ProcessedDatabase.swift): its contexts, one resident .diagonal matrix per context, the entry
    identifiers and metadata."""

    def __init__(self, contexts, plaintextMatrices, entryIds, entryMetadatas, serverConfig: ServerConfig):
        self.contexts, self.plaintextMatrices = list(contexts), list(plaintextMatrices)
        self.entryIds, self.entryMetadatas, self.serverConfig = list(entryIds), list(entryMetadatas), serverConfig

    @classmethod
    def processOnDevice(cls, database: Database, serverConfig: ServerConfig, contexts) -> "ProcessedDatabase":
        """Database.process (ProcessedDatabase.swift:194-229) on the device (hecuda_pnns_matrices_create_from_vectors):
        the float rows cross PCIe once, are normalised, scaled and rounded once, and packed into one resident Eval
        matrix per context, reduced mod t when there are several."""
        _check_metric(serverConfig.distanceMetric)
        serverConfig.validateContexts(contexts)
        if not database.rows:
            raise PnnsError("emptyDatabase")
        vectors = _float_rows([row.vector for row in database.rows])
        rows, cols = vectors.shape
        dims = MatrixDimensions(rows, cols)
        bsgs = serverConfig.babyStepGiantStep
        handles = (C.c_void_p * len(contexts))()
        ctxs = (C.c_void_p * len(contexts))(*[c._h.value for c in contexts])
        _check(load_library().hecuda_pnns_matrices_create_from_vectors(
            ctxs, len(contexts), vectors.ctypes.data_as(C.c_void_p), rows, cols, serverConfig.scalingFactor, bsgs.babyStep,
            bsgs.giantStep, handles))
        matrices = []
        for ctx, h in zip(contexts, handles):
            m = PlaintextMatrix.__new__(PlaintextMatrix)
            m.context, m.dimensions, m.babyStepGiantStep, m._h = ctx, dims, bsgs, C.c_void_p(h)
            m.resultCiphertextCount = -(-rows // ctx.degree)
            matrices.append(m)
        has_metadata = any(len(row.entryMetadata) for row in database.rows)
        return cls(contexts, matrices, [row.entryId for row in database.rows],
                   [bytes(row.entryMetadata) for row in database.rows] if has_metadata else [], serverConfig)

    def _entries(self):
        ids = np.ascontiguousarray(np.asarray(self.entryIds, dtype=np.uint64)).reshape(-1)
        meta = [bytes(m) for m in self.entryMetadatas]
        offsets = np.zeros(len(meta) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(m) for m in meta], dtype=np.uint64)
        blob = np.frombuffer(b"".join(meta) or b"\0", dtype=np.uint8)
        config = _config_struct(self.serverConfig.clientConfig, self.serverConfig.babyStepGiantStep)
        handles = (C.c_void_p * len(self.plaintextMatrices))(*[m._h.value for m in self.plaintextMatrices])
        return (handles, len(self.plaintextMatrices), _ptr(ids) if ids.size else None, ids.size, _ptr(blob), _ptr(offsets),
                len(meta), C.byref(config)), (ids, blob, offsets, config)

    def serializationByteCount(self) -> int:
        """The byte count of serialize()."""
        args, keep = self._entries()
        size = C.c_uint64(0)
        _check(load_library().hecuda_pnns_database_serialized_byte_count(*args, C.byref(size)))
        return size.value

    def _serialize_into(self, out: np.ndarray):
        args, keep = self._entries()
        written = C.c_uint64(0)
        _check(load_library().hecuda_pnns_database_serialize(*args, _ptr(out), out.size, C.byref(written)))

    def serialize(self) -> bytes:
        """ProcessedDatabase.serialize().proto().serializedData() (ProcessedDatabase.swift:81-88): the
        SerializedProcessedDatabase protobuf message, byte for byte as SwiftProtobuf writes it.  The plaintexts are
        packed on the device with their framing (hecuda_pnns_database_serialize)."""
        out = np.empty(self.serializationByteCount(), dtype=np.uint8)
        self._serialize_into(out)
        return out.tobytes()

    def save(self, path) -> None:
        """serialize(), written straight into the file's pages (the reference's `.binpb` file)."""
        import os
        out = np.memmap(path, dtype=np.uint8, mode="w+", shape=(self.serializationByteCount(),))
        try:
            self._serialize_into(out)
            out.flush()
        except Exception:
            del out
            os.remove(path)
            raise

    @classmethod
    def load(cls, source, contexts=None) -> "ProcessedDatabase":
        """ProcessedDatabase(from:contexts:) (ProcessedDatabase.swift:56-75) of a SerializedProcessedDatabase, unpacked on
        the device (hecuda_pnns_matrices_create_serialized).  source: bytes, a uint8 array, or a path, which is mapped
        with np.memmap.  Without contexts, one Context per encryption parameters set of the config is created.  Raises
        HeError with the reference's error names; also where the reference would accept a residue >= its modulus or
        trap on a truncated buffer."""
        from .pir import _source_bytes
        data = _source_bytes(source)
        buf = data if data.size else np.zeros(1, dtype=np.uint8)
        lib = load_library()
        config = _ConfigStruct()
        matrices, rows, cols, id_count, meta_count = C.c_int32(0), C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
        meta_bytes = C.c_uint64(0)
        _check(lib.hecuda_pnns_database_describe(_ptr(buf), data.size, C.byref(config), C.byref(matrices), C.byref(rows),
                                                 C.byref(cols), C.byref(id_count), C.byref(meta_count), C.byref(meta_bytes)))
        serverConfig = _server_config(config)
        if contexts is None:
            p = serverConfig.encryptionParameters[0]
            contexts = [Context(p.polyDegree, list(p.coefficientModuli), t) for t in serverConfig.plaintextModuli]
        contexts = list(contexts)
        serverConfig.validateContexts(contexts)
        handles = (C.c_void_p * len(contexts))()
        ctxs = (C.c_void_p * len(contexts))(*[c._h.value for c in contexts])
        _check(lib.hecuda_pnns_matrices_create_serialized(ctxs, len(contexts), _ptr(buf), data.size, handles))
        ids = np.empty(max(1, id_count.value), dtype=np.uint64)
        blob = np.empty(max(1, meta_bytes.value), dtype=np.uint8)
        offsets = np.empty(meta_count.value + 1, dtype=np.uint64)
        _check(lib.hecuda_pnns_database_entries(_ptr(buf), data.size, _ptr(ids), ids.size, _ptr(blob), blob.size,
                                                _ptr(offsets), offsets.size))
        dims = MatrixDimensions(rows.value, cols.value)
        out = []
        for ctx, h in zip(contexts, handles):
            m = PlaintextMatrix.__new__(PlaintextMatrix)
            m.context, m.dimensions, m.babyStepGiantStep, m._h = ctx, dims, serverConfig.babyStepGiantStep, C.c_void_p(h)
            m.resultCiphertextCount = -(-rows.value // ctx.degree)
            out.append(m)
        metadatas = [blob[int(offsets[k]):int(offsets[k + 1])].tobytes() for k in range(meta_count.value)]
        return cls(contexts, out, [int(v) for v in ids[:id_count.value]], metadatas, serverConfig)

    def validate(self, queryVectors, trials: int = 1) -> ValidationResult:
        """ProcessedDatabase.validate (ProcessedDatabase.swift:91-143), every step on the device."""
        import time
        from . import Bfv
        if trials <= 0:
            raise PnnsError(f"validationError(Invalid trialsPerShard: {trials})")
        v = _float_rows(queryVectors)
        if v.shape[1] != self.serverConfig.vectorDimension:
            raise PnnsError(f"validationError(Wrong vector dimension {v.shape[1]}, expected {self.serverConfig.vectorDimension})")
        server = Server(self)
        client = Client(self.serverConfig.clientConfig, self.contexts)
        first_key = first_query = response = distances = None
        min_budget, times = math.inf, []
        for trial in range(trials):
            secret_key = client.generateSecretKey()
            key = client.generateEvaluationKey(secret_key)
            query = client.generateQuery(v, secret_key)
            start = time.perf_counter()
            response = server.computeResponse(query, key)
            times.append(time.perf_counter() - start)
            budget = response.noiseBudget(self.contexts, secret_key)
            if budget < Bfv.minNoiseBudget:
                raise PnnsError("validationError(Insufficient noise budget)")
            decrypted = client.decrypt(response, secret_key)
            min_budget = min(min_budget, budget)
            if trial == 0:
                first_key, first_query, distances = key, query, decrypted
            else:
                key.close()
        return ValidationResult(first_key, first_query, response, distances, min_budget, times)

    def close(self):
        for m in self.plaintextMatrices:
            m.close()


class Server:
    """Server (Server.swift:19-89) over a processed database, one matrix per plaintext modulus."""

    def __init__(self, database: ProcessedDatabase):
        _check_metric(database.serverConfig.distanceMetric)
        self.database = database

    @property
    def contexts(self):
        return self.database.contexts

    def _check(self, query: Query):
        expected = len(self.database.plaintextMatrices)
        if len(query.ciphertextMatrices) != expected:
            raise PnnsError(f"invalidQuery(wrongCiphertextMatrixCount(got: {len(query.ciphertextMatrices)}, expected: {expected}))")

    def computeResponse(self, query: Query, evaluationKey: EvaluationKey) -> Response:
        """Server.computeResponse (Server.swift:61-88): mulTranspose(matrix:) and modSwitchDownToSingle per matrix, the
        key copied to contexts 1 and up (EvaluationKey.forContext)."""
        return self.computeResponses([query], [evaluationKey])[0]

    def computeResponses(self, queries, evaluationKeys) -> list:
        """computeResponse for many clients, each with its own key: one PlaintextMatrix.computeResponses call (or its
        wire form for wire queries) per matrix."""
        queries, keys = list(queries), list(evaluationKeys)
        for q in queries:
            self._check(q)
        if not queries or len(queries) != len(keys):
            raise PnnsError("one evaluation key per query")
        dims = queries[0].dimensions
        if any(q.dimensions != dims or q.wire != queries[0].wire for q in queries):
            raise PnnsError("every query must have the same dimensions and form")
        per_matrix = []
        for k, m in enumerate(self.database.plaintextMatrices):
            ctx_keys = [key.forContext(m.context) for key in keys]
            if queries[0].wire:
                poly0 = np.stack([q.ciphertextMatrices[k][0] for q in queries])
                seeds = np.stack([q.ciphertextMatrices[k][1] for q in queries])
                replies, skips = PnnsWire.computeResponses(m, poly0, seeds, dims, ctx_keys)
                per_matrix.append([(replies[c], skips) for c in range(len(queries))])
            else:
                cts = np.stack([q.ciphertextMatrices[k] for q in queries])
                if len(queries) == 1:
                    replies = m.mulTransposeMatrix(cts[0], dims, ctx_keys[0], modSwitchDownToSingle=True)[None]
                else:
                    replies = m.computeResponses(cts, dims, ctx_keys)
                per_matrix.append([replies[c] for c in range(len(queries))])
        out_dims = MatrixDimensions(self.database.plaintextMatrices[0].dimensions.rowCount, dims.rowCount)
        return [Response([per_matrix[k][c] for k in range(len(per_matrix))], out_dims, list(self.database.entryIds),
                         list(self.database.entryMetadatas)) for c in range(len(queries))]

    def computeResponsesProto(self, messages, evaluationKeys) -> list:
        """computeResponses with protobuf messages (hecuda_pnns_compute_response_clients_proto): one
        api.pnns.v1.PNNSRequest per client in (only its query matrices are read; .seeded or .full ciphertexts), one
        api.pnns.v1.PNNSShardResponse per client out, with the database's entry ids and metadata.  The query plan is
        derived in the library from the message's shape.  Keys loaded on contexts[0] (e.g. by
        EvaluationKey.fromProtoMany) serve every plaintext modulus as they are, with no forContext copies."""
        keys = list(evaluationKeys)
        ptrs, counts, keep = _message_buffers(messages)
        if not keys or len(keep) != len(keys):
            raise PnnsError(f"computeResponsesProto: {len(keep)} messages for {len(keys)} evaluation keys")
        db = self.database
        K = len(db.plaintextMatrices)
        ctxs = (C.c_void_p * K)(*[m.context._h.value for m in db.plaintextMatrices])
        handles = (C.c_void_p * K)(*[m._h.value for m in db.plaintextMatrices])
        ids = np.ascontiguousarray(np.asarray(db.entryIds, dtype=np.uint64)).reshape(-1)
        meta = [bytes(m) for m in db.entryMetadatas]
        offsets = np.zeros(len(meta) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(m) for m in meta], dtype=np.uint64)
        blob = np.frombuffer(b"".join(meta) or b"\0", dtype=np.uint8)
        entries = (_ptr(ids) if ids.size else None, ids.size, blob.ctypes.data_as(C.c_void_p), _ptr(offsets), len(meta))
        lib = load_library()
        first = PnnsRequest.fields(bytes(keep[0][:int(counts[0])]))
        size = C.c_uint64(0)
        _check(lib.hecuda_pnns_shard_response_byte_count(ctxs, K, handles, max(1, first["queryRowCount"]), *entries,
                                                         C.byref(size)))
        out = np.empty((len(keys), size.value), dtype=np.uint8)
        key_handles = (C.c_void_p * len(keys))(*[k._h.value if hasattr(k._h, "value") else k._h for k in keys])
        _check(lib.hecuda_pnns_compute_response_clients_proto(ctxs, K, key_handles, len(keys), handles, ptrs,
                                                              counts.ctypes.data_as(C.c_void_p), *entries,
                                                              out.ctypes.data_as(C.c_void_p)))
        return [row.tobytes() for row in out]
