"""hecuda.simple_pir -- the reference's SimplePIR server over libhecuda.

Names follow Sources/PrivateInformationRetrieval/SimplePir/:

    SimplePirEncryptionParams, SimplePirParameters          SimplePir.swift:19-160
    SimplePirServer.computingParams / process               SimplePir+Database.swift:208-290
    SimplePirServer(processedDatabase:hint:params:)         SimplePir+Server.swift:24-29
    SimplePirServer.computeResponse                         SimplePir+Server.swift:31-38
    Array2d.save / init(from:)                              SimplePir+Database.swift:36-121

The processed database stays on the device as u8 digit planes; responses are integer tensor-core products there.
`scalar` is the reference's Scalar type: np.uint32 (UInt32) or np.uint64 (UInt64).
"""
from __future__ import annotations

import ctypes as C
import math
import secrets
import struct
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _check, _ptr, load_library
from .pir import PirError

SEED_BYTES = 32  # NistAes128Ctr.SeedCount

# EncryptionParameters.maxLog2CoefficientModulus (EncryptionParameters.swift:192-219) for .quantum128: the largest
# log2 of the coefficient modulus per degree, for error standard deviation 3.2 and (at N = 2048 only) 6.4
_MAX_LOG2_Q_STDDEV32 = {1 << 10: 21, 1 << 11: 41, 1 << 12: 83, 1 << 13: 165, 1 << 14: 330, 1 << 15: 660}
_MAX_LOG2_Q_STDDEV64 = {1 << 11: 42}


class _Params(C.Structure):  # hecuda_simple_pir_params
    _fields_ = [("plaintext_modulus_bits", C.c_int32), ("ciphertext_modulus_bits", C.c_int32),
                ("lattice_dimension", C.c_int64), ("entry_size", C.c_int64), ("entries_per_column", C.c_int64),
                ("chunks_per_entry", C.c_int64), ("database_columns", C.c_int64), ("word_bits", C.c_int32)]


@dataclass(frozen=True)
class SimplePirEncryptionParams:
    """errorStdDev is 3.2 (.stdDev32) or 6.4 (.stdDev64); securityLevel "quantum128" or "unchecked"."""
    plaintextModulusBits: int
    ciphertextModulusBits: int
    latticeDimension: int
    errorStdDev: float = 3.2
    securityLevel: str = "quantum128"

    def __post_init__(self):
        n = self.latticeDimension
        if n < 1 or n & (n - 1):
            raise PirError(f"invalidEncryptionParameters: SimplePir latticeDimension={n} is not a power of 2")
        if self.errorStdDev not in (3.2, 6.4):
            raise PirError(f"invalidEncryptionParameters: errorStdDev must be 3.2 (.stdDev32) or 6.4 (.stdDev64), "
                           f"got {self.errorStdDev}")
        if self.ciphertextModulusBits <= self.plaintextModulusBits:
            raise PirError("invalidEncryptionParameters: SimplePir ciphertextModulusBits must be > plaintextModulusBits")
        if self.securityLevel == "unchecked":
            return
        table = _MAX_LOG2_Q_STDDEV64 if self.errorStdDev == 6.4 else _MAX_LOG2_Q_STDDEV32
        if n not in table:
            raise PirError(f"invalidEncryptionParameters: no quantum128 bound for latticeDimension={n}, "
                           f"errorStdDev={self.errorStdDev}")
        if self.ciphertextModulusBits > table[n]:
            raise PirError(f"insecureEncryptionParameters: ciphertextModulusBits={self.ciphertextModulusBits} "
                           f"exceeds {table[n]} for latticeDimension={n}")


def _coeff_count(byte_count: int, bits: int) -> int:  # CoefficientPacking.bytesToCoefficientsCoeffCount(decode: false)
    return -(-byte_count * 8 // bits)


@dataclass(frozen=True)
class SimplePirParameters:
    encryptionParams: SimplePirEncryptionParams
    entrySizeInBytes: int
    entriesPerColumn: int
    chunksPerEntry: int
    databaseColumns: int
    seed: bytes = field(default=b"\0" * SEED_BYTES)

    def __post_init__(self):
        if not (self.entriesPerColumn == 1 or self.chunksPerEntry == 1):
            raise PirError("SimplePirParameters: entriesPerColumn == 1 || chunksPerEntry == 1")

    plaintextModulusBits = property(lambda self: self.encryptionParams.plaintextModulusBits)
    ciphertextModulusBits = property(lambda self: self.encryptionParams.ciphertextModulusBits)
    latticeDimension = property(lambda self: self.encryptionParams.latticeDimension)

    @property
    def entrySizeInScalar(self) -> int:
        return _coeff_count(self.entrySizeInBytes, self.plaintextModulusBits)

    @property
    def chunkSize(self) -> int:
        return -(-self.entrySizeInScalar // self.chunksPerEntry)

    @property
    def columnSize(self) -> int:
        return self.entriesPerColumn * self.entrySizeInScalar if self.chunksPerEntry == 1 else self.chunkSize

    @property
    def aPolyCount(self) -> int:
        return -(-self.databaseColumns // self.latticeDimension)

    @staticmethod
    def computingParams(encryptionParams: SimplePirEncryptionParams, entryCount: int, entrySizeInBytes: int,
                        seed: Optional[bytes] = None) -> "SimplePirParameters":
        """SimplePirServerProtocol.computingParams (SimplePir+Database.swift:208-243).  Swift's .rounded() rounds halves
        away from zero (floor(x + 0.5) here, every operand being >= 0), and chunksPerEntry truncates."""
        scalars = _coeff_count(entrySizeInBytes, encryptionParams.plaintextModulusBits)
        ideal_column = min(math.floor(math.sqrt(float(entryCount * scalars)) + 0.5), scalars)
        entries_per_column = max(math.floor(float(ideal_column) / float(scalars) + 0.5), 1)
        chunks_per_entry = max(int(float(scalars) / float(ideal_column)), 1)
        columns = entryCount * chunks_per_entry if entries_per_column == 1 else max(-(-entryCount // entries_per_column), 1)
        return SimplePirParameters(encryptionParams, entrySizeInBytes, entries_per_column, chunks_per_entry, columns,
                                   secrets.token_bytes(SEED_BYTES) if seed is None else bytes(seed))

    def _c(self, word_bits: int) -> _Params:
        return _Params(self.plaintextModulusBits, self.ciphertextModulusBits, self.latticeDimension, self.entrySizeInBytes,
                       self.entriesPerColumn, self.chunksPerEntry, self.databaseColumns, word_bits)


def _word_bits(scalar) -> int:
    scalar = np.dtype(scalar)
    if scalar not in (np.dtype(np.uint32), np.dtype(np.uint64)):
        raise PirError("SimplePir scalar must be np.uint32 or np.uint64")
    return scalar.itemsize * 8


def save_array2d(array: np.ndarray, path: str):
    """Array2d.save(to:): u32 LE row and column counts, then the scalars little-endian."""
    array = np.asarray(array)
    with open(path, "wb") as f:
        f.write(struct.pack("<II", array.shape[0], array.shape[1]))
        f.write(np.ascontiguousarray(array, dtype=array.dtype.newbyteorder("<")).tobytes())


def load_array2d(path: str, scalar=np.uint64) -> np.ndarray:
    """Array2d(from:); PirError.corruptedData on a truncated file."""
    dtype = np.dtype(scalar).newbyteorder("<")
    with open(path, "rb") as f:
        header = f.read(8)
        if len(header) < 8:
            raise PirError("corruptedData: Unexpected EOF")
        rows, cols = struct.unpack("<II", header)
        if rows * cols >= 16_000_000_000:
            raise PirError(f"corruptedData: Database is unreasonably large: {rows} x {cols}")
        body = f.read(rows * cols * dtype.itemsize)
    if len(body) < rows * cols * dtype.itemsize:
        raise PirError("corruptedData: Unexpected EOF")
    return np.frombuffer(body, dtype=dtype).astype(np.dtype(scalar)).reshape(rows, cols)


class SimplePirDatabase:
    """The processed database (columnSize x databaseColumns), resident on the device."""

    def __init__(self, handle, params: SimplePirParameters, scalar):
        self._h, self.params, self.scalar = handle, params, np.dtype(scalar)

    @staticmethod
    def create(processedDatabase, params: SimplePirParameters, scalar=np.uint64) -> "SimplePirDatabase":
        bits = _word_bits(scalar)
        matrix = np.ascontiguousarray(np.asarray(processedDatabase, dtype=scalar))
        if matrix.shape != (params.columnSize, params.databaseColumns):
            raise PirError(f"processed database must be {params.columnSize} x {params.databaseColumns}, got {matrix.shape}")
        h = C.c_void_p()
        cp = params._c(bits)
        _check(load_library().hecuda_simple_pir_database_create(_ptr(matrix), C.byref(cp), C.byref(h)))
        return SimplePirDatabase(h, params, scalar)

    def export(self) -> np.ndarray:
        out = np.empty((self.params.columnSize, self.params.databaseColumns), dtype=self.scalar)
        _check(load_library().hecuda_simple_pir_database_export(self._h, _ptr(out)))
        return out

    def save(self, path: str):
        save_array2d(self.export(), path)

    @staticmethod
    def load(path: str, params: SimplePirParameters, scalar=np.uint64) -> "SimplePirDatabase":
        return SimplePirDatabase.create(load_array2d(path, scalar), params, scalar)

    def close(self):
        if self._h is not None:
            load_library().hecuda_simple_pir_database_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class SimplePIRProcessDatabaseResults:
    database: SimplePirDatabase
    hint: np.ndarray
    params: SimplePirParameters


class SimplePirServer:
    """SimplePirServer<Scalar>: construct from a processed database (host matrix or SimplePirDatabase), its hint and
    params; SimplePirServer.process builds all three from raw entries on the device."""

    def __init__(self, processedDatabase, hint, params: SimplePirParameters, scalar=np.uint64):
        self.scalar = np.dtype(scalar)
        _word_bits(self.scalar)
        self.database = (processedDatabase if isinstance(processedDatabase, SimplePirDatabase)
                         else SimplePirDatabase.create(processedDatabase, params, self.scalar))
        self.hint = np.asarray(hint, dtype=self.scalar)
        self.params = params

    @staticmethod
    def process(database, encryptionParams: SimplePirEncryptionParams, seed: Optional[bytes] = None,
                scalar=np.uint64) -> SimplePIRProcessDatabaseResults:
        """database: entryCount x entrySizeInBytes uint8 (RawDatabase = Array2d<UInt8>)."""
        bits = _word_bits(scalar)
        raw = np.ascontiguousarray(np.asarray(database, dtype=np.uint8))
        if raw.ndim != 2 or raw.shape[0] < 1 or raw.shape[1] < 1:
            raise PirError("SimplePir database must be a non-empty entryCount x entrySizeInBytes byte matrix")
        params = SimplePirParameters.computingParams(encryptionParams, raw.shape[0], raw.shape[1], seed)
        if len(params.seed) != SEED_BYTES:
            raise PirError(f"seed must be {SEED_BYTES} bytes")
        hint = np.empty((params.columnSize, params.latticeDimension), dtype=scalar)
        seed_buf = np.frombuffer(params.seed, dtype=np.uint8).copy()
        h = C.c_void_p()
        cp = params._c(bits)
        _check(load_library().hecuda_simple_pir_process(_ptr(raw), raw.shape[0], C.byref(cp), _ptr(seed_buf), _ptr(hint),
                                                        C.byref(h)))
        return SimplePIRProcessDatabaseResults(SimplePirDatabase(h, params, scalar), hint, params)

    def _requests(self, requests) -> np.ndarray:
        r = np.ascontiguousarray(np.asarray(requests, dtype=self.scalar))
        if r.ndim == 2:
            r = r[None]
        if r.ndim != 3 or r.shape[1:] != (self.params.chunksPerEntry, self.params.databaseColumns):
            raise PirError(f"request must be {self.params.chunksPerEntry} x {self.params.databaseColumns}, got "
                           f"{np.asarray(requests).shape}")
        return r

    def computeResponses(self, requests: Sequence) -> np.ndarray:
        """Responses to many requests in one device pass: count x chunksPerEntry x columnSize."""
        r = self._requests(np.stack([np.asarray(x, dtype=self.scalar) for x in requests]) if isinstance(requests, list)
                           else requests)
        out = np.empty((r.shape[0], self.params.chunksPerEntry, self.params.columnSize), dtype=self.scalar)
        _check(load_library().hecuda_simple_pir_compute_response(self.database._h, _ptr(r), r.shape[0], _ptr(out)))
        return out

    def computeResponse(self, requests) -> np.ndarray:
        """computeResponse(to:): chunksPerEntry x K request words -> chunksPerEntry x columnSize."""
        return self.computeResponses(self._requests(requests))[0]

    def computeResponsesDevice(self, requests_ptr: int, count: int, responses_ptr: int, stream: int = 0):
        """Device buffers (torch data_ptr()): enqueue on `stream` without synchronising."""
        _check(load_library().hecuda_simple_pir_compute_response_device(self.database._h, C.c_void_p(requests_ptr), count,
                                                                        C.c_void_p(responses_ptr), C.c_void_p(stream)))
