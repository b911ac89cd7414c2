"""hecuda.symmetric_pir -- the reference's symmetric PIR configuration and OPRF over libhecuda.

Names follow Sources/PrivateInformationRetrieval/SymmetricPir/SymmetricPirDatabase.swift:

    SymmetricPirConfigType, SymmetricPirClientConfig, SymmetricPirConfig   :21-184
    KeywordDatabase.symmetricPIRProcess                                    :186-211 (hecuda.keyword_pir)

The OPRF is RFC 9497 in VOPRF mode over P384-SHA384 (swift-crypto's P384._VOPRF), evaluated on the device one thread
per row; the rows' AES-GCM-192 sealing runs there too.
"""
from __future__ import annotations

import enum
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

from . import _check, _ptr, load_library
from .pir import PirError

OPRF_KEY_BYTES, OPRF_ELEMENT_BYTES, OPRF_OUTPUT_BYTES = 48, 49, 48  # HECUDA_OPRF_*


def _concatenate(blobs: Sequence[bytes]):
    blobs = [bytes(b) for b in blobs]
    offsets = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    data = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)
    return data, offsets


def _key(secretKey: bytes) -> np.ndarray:
    key = np.frombuffer(bytes(secretKey), dtype=np.uint8)
    if key.size != OPRF_KEY_BYTES:
        raise PirError(f"invalidOPRFKeySize({key.size}, expectedSize: {OPRF_KEY_BYTES})")
    return key


class SymmetricPirConfigType(enum.Enum):
    """SymmetricPirConfigType (:21-65)."""

    OPRF_P384_AES_GCM_192_NONCE_96_TAG_128 = "OPRF_P384_AES_GCM_192_NONCE_96_TAG_128"

    @property
    def oprfKeySize(self) -> int:
        return 48

    @property
    def oprfOutputSize(self) -> int:
        return 48

    @property
    def obliviousKeywordSize(self) -> int:
        return 16

    @property
    def entryEncryptionKeySize(self) -> int:
        return 24

    @property
    def nonceSize(self) -> int:
        return 12

    @property
    def tagSize(self) -> int:
        return 16


@dataclass(frozen=True)
class SymmetricPirClientConfig:
    """SymmetricPirClientConfig (:79-95)."""

    serverPublicKey: bytes
    configType: SymmetricPirConfigType = SymmetricPirConfigType.OPRF_P384_AES_GCM_192_NONCE_96_TAG_128


class SymmetricPirConfig:
    """SymmetricPirConfig (:151-184).  The key is kept as bytes; repr never shows it."""

    def __init__(self, oprfSecretKey: bytes,
                 configType: SymmetricPirConfigType = SymmetricPirConfigType.OPRF_P384_AES_GCM_192_NONCE_96_TAG_128):
        oprfSecretKey = bytes(oprfSecretKey)
        if len(oprfSecretKey) != configType.oprfKeySize:
            raise PirError(f"invalidOPRFKeySize({len(oprfSecretKey)}, expectedSize: {configType.oprfKeySize})")
        self.oprfSecretKey, self.configType = oprfSecretKey, configType

    def __repr__(self) -> str:
        return f"SymmetricPirConfig(oprfSecretKey: ****, configType: {self.configType.value})"

    def clientConfig(self) -> SymmetricPirClientConfig:
        """clientConfig() (:176-183): the OPRF public key k G, compressed."""
        return SymmetricPirClientConfig(Oprf.publicKey(self.oprfSecretKey), self.configType)


class Oprf:
    """OprfPrivateKey (swift-crypto P384._VOPRF.PrivateKey) on the device."""

    @staticmethod
    def publicKey(secretKey: bytes) -> bytes:
        out = np.zeros(OPRF_ELEMENT_BYTES, dtype=np.uint8)
        _check(load_library().hecuda_oprf_public_key(_ptr(_key(secretKey)), _ptr(out)))
        return out.tobytes()

    @staticmethod
    def evaluate(secretKey: bytes, inputs: Sequence[bytes]) -> np.ndarray:
        """evaluate(_:) of every input (RFC 9497 Evaluate) -> (count, 48) uint8."""
        data, offsets = _concatenate(inputs)
        count = len(offsets) - 1
        out = np.zeros((max(count, 1), OPRF_OUTPUT_BYTES), dtype=np.uint8)
        _check(load_library().hecuda_oprf_evaluate(_ptr(_key(secretKey)), _ptr(data), _ptr(offsets), count, _ptr(out)))
        return out[:count]


def symmetricPIRProcess(database: Sequence[Tuple[bytes, bytes]], config: SymmetricPirConfig) -> List[Tuple[bytes, bytes]]:
    """KeywordDatabase.symmetricPIRProcess(database:config:) (:193-211): (keyword, value) -> (h[0:16],
    AES-GCM-192-seal(value) as ciphertext || tag) with h the keyword's OPRF output, every row on the device."""
    if config.configType is not SymmetricPirConfigType.OPRF_P384_AES_GCM_192_NONCE_96_TAG_128:
        raise PirError(f"invalidSymmetricPirConfig(symmetricPirConfig: {config})")
    rows = [(bytes(k), bytes(v)) for k, v in database]
    keywords, koff = _concatenate([k for k, _ in rows])
    values, voff = _concatenate([v for _, v in rows])
    count = len(rows)
    tag = config.configType.tagSize
    keywords_out = np.zeros(max(count, 1) * 16, dtype=np.uint8)
    values_out = np.zeros(max(int(voff[-1]) + tag * count, 1), dtype=np.uint8)
    _check(load_library().hecuda_symmetric_pir_process(_ptr(_key(config.oprfSecretKey)), _ptr(keywords), _ptr(koff),
                                                       _ptr(values), _ptr(voff), count, _ptr(keywords_out),
                                                       _ptr(values_out)))
    kw, raw = keywords_out.tobytes(), values_out.tobytes()
    return [(kw[16 * i:16 * (i + 1)], raw[int(voff[i]) + tag * i:int(voff[i + 1]) + tag * (i + 1)]) for i in range(count)]
