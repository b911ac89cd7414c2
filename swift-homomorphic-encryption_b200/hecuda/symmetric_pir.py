"""hecuda.symmetric_pir -- the reference's symmetric PIR configuration and OPRF over libhecuda.

Names follow Sources/PrivateInformationRetrieval/SymmetricPir/SymmetricPirDatabase.swift:

    SymmetricPirConfigType, SymmetricPirClientConfig, SymmetricPirConfig   :21-184
    KeywordDatabase.symmetricPIRProcess                                    :186-211 (hecuda.keyword_pir)
    OprfServer                        SymmetricPir/SymmetricPirProtocol.swift:39-59
    OprfClient, ParsedOprfOutput      SymmetricPir/SymmetricPirProtocol.swift:62-133
    OprfQueryContext (.query)         SymmetricPir/SymmetricPirProtocol.swift:20-36

The OPRF is RFC 9497 in VOPRF mode over P384-SHA384 (swift-crypto's P384._VOPRF), evaluated on the device one thread
per row; the rows' AES-GCM-192 sealing runs there too, and so do the server's answers to clients' blinded queries and
the client's blinding, proof verification, finalization and opening of retrieved entries.
"""
from __future__ import annotations

import enum
import secrets
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _check, _ptr, load_library
from .pir import PirError

OPRF_KEY_BYTES, OPRF_ELEMENT_BYTES, OPRF_OUTPUT_BYTES = 48, 49, 48  # HECUDA_OPRF_*
OPRF_RESPONSE_BYTES, OPRF_SEED_BYTES = 145, 32
# the order n of P-384's group: blinds are drawn from [1, n - 1]
P384_ORDER = 0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973


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


class OprfServer:
    """OprfServer (SymmetricPirProtocol.swift:39-59): answers clients' blinded OPRF queries on the device with RFC 9497
    BlindEvaluate and its DLEQ proof.  A response is the 145 bytes swift-crypto's BlindEvaluation(rawRepresentation:)
    takes: the evaluated element, then the proof's c and s.

    `seed` (32 bytes, random by default) hedges the proof nonce, which is derived from the key and the query: the
    same seed gives the same response, and no seed can make two different challenges share a nonce."""

    def __init__(self, symmetricPirConfig: SymmetricPirConfig):
        if symmetricPirConfig.configType is not SymmetricPirConfigType.OPRF_P384_AES_GCM_192_NONCE_96_TAG_128:
            raise PirError(f"invalidSymmetricPirConfig(symmetricPirConfig: {symmetricPirConfig})")
        self._key = _key(symmetricPirConfig.oprfSecretKey)

    def computeResponse(self, query: bytes, seed: Optional[bytes] = None) -> bytes:
        """computeResponse(query:): PirError when the query is not a valid compressed P-384 point."""
        response = self.computeResponses([query], seed)[0]
        if response is None:
            raise PirError("invalidOprfQuery: not a valid SEC1-compressed P-384 element")
        return response

    def computeResponses(self, queries: Sequence[bytes], seed: Optional[bytes] = None) -> List[Optional[bytes]]:
        """One response per query in one device call; None where a query is invalid, including a wrong length."""
        seed = secrets.token_bytes(OPRF_SEED_BYTES) if seed is None else bytes(seed)
        if len(seed) != OPRF_SEED_BYTES:
            raise PirError(f"OPRF proof seed must be {OPRF_SEED_BYTES} bytes, got {len(seed)}")
        queries = [bytes(q) for q in queries]
        sized = [i for i, q in enumerate(queries) if len(q) == OPRF_ELEMENT_BYTES]
        count = len(sized)
        blinded = np.frombuffer(b"".join(queries[i] for i in sized) or b"\0", dtype=np.uint8)
        responses = np.zeros((max(count, 1), OPRF_RESPONSE_BYTES), dtype=np.uint8)
        status = np.ones(max(count, 1), dtype=np.uint8)
        _check(load_library().hecuda_oprf_blind_evaluate(_ptr(self._key), _ptr(blinded), count,
                                                         _ptr(np.frombuffer(seed, dtype=np.uint8)), _ptr(responses),
                                                         _ptr(status)))
        out: List[Optional[bytes]] = [None] * len(queries)
        for j, i in enumerate(sized):
            if status[j] == 0:
                out[i] = responses[j].tobytes()
        return out


@dataclass(frozen=True, repr=False)
class OprfQueryContext:
    """OprfQueryContext (swift-crypto's P384._VOPRF.BlindedInput): the keyword, its secret blind r and the query
    Ser(r HashToGroup(keyword)) to send to the server (the `query` extension, SymmetricPirProtocol.swift:31-36).  repr
    never shows the blind."""

    keyword: bytes
    blind: int
    query: bytes

    def __repr__(self) -> str:
        return f"OprfQueryContext(keyword: {self.keyword!r}, blind: ****, query: {self.query.hex()})"


@dataclass(frozen=True, repr=False)
class ParsedOprfOutput:
    """OprfClient.ParsedOprfOutput (:64-82): the finalized OPRF output split into the oblivious keyword (its first 16
    bytes), the entry's nonce (its first 12) and the entry's AES key (its last 24).  repr never shows the key."""

    obliviousKeyword: bytes
    nonce: bytes
    secretKey: bytes

    @classmethod
    def fromOprfOutput(cls, oprfOutput: bytes, configType: SymmetricPirConfigType) -> "ParsedOprfOutput":
        oprfOutput = bytes(oprfOutput)
        return cls(oprfOutput[:configType.obliviousKeywordSize], oprfOutput[:configType.nonceSize],
                   oprfOutput[len(oprfOutput) - configType.entryEncryptionKeySize:])

    def __repr__(self) -> str:
        return f"ParsedOprfOutput(obliviousKeyword: {self.obliviousKeyword.hex()}, nonce: {self.nonce.hex()}, secretKey: ****)"


class OprfClient:
    """OprfClient (SymmetricPirProtocol.swift:62-133) on the device: blinding, the server's proof check, unblinding and
    finalization, and the AES-GCM open of retrieved entries, each one device call for a whole list."""

    def __init__(self, symmetricPirClientConfig: SymmetricPirClientConfig):
        config = symmetricPirClientConfig
        if config.configType is not SymmetricPirConfigType.OPRF_P384_AES_GCM_192_NONCE_96_TAG_128:
            raise PirError(f"invalidSymmetricPirConfig(symmetricPirConfig: {config})")
        key = bytes(config.serverPublicKey)
        if len(key) != OPRF_ELEMENT_BYTES:
            raise PirError(f"invalid OPRF public key: {len(key)} bytes, expected {OPRF_ELEMENT_BYTES}")
        self._publicKey = np.frombuffer(key, dtype=np.uint8)
        self.configType = config.configType
        lib = load_library()
        none = np.zeros(1, dtype=np.uint64)  # a finalize of no queries checks the key and launches nothing
        if lib.hecuda_oprf_finalize(_ptr(self._publicKey), _ptr(none), _ptr(none), 0, _ptr(none), _ptr(none),
                                    _ptr(none), _ptr(none), _ptr(none)) != 0:
            raise PirError("invalid OPRF public key: " + (lib.hecuda_last_error() or b"").decode())

    def queryContext(self, keyword: bytes) -> OprfQueryContext:
        """queryContext(at:) (:98-104) with a fresh random blind."""
        return self.queryContexts([keyword])[0]

    def queryContexts(self, keywords: Sequence[bytes], blinds: Optional[Sequence[int]] = None) -> List[OprfQueryContext]:
        """One context per keyword in one device call.  `blinds` (integers in [1, n - 1]) defaults to fresh draws from
        `secrets`; PirError for a blind outside that range."""
        keywords = [bytes(k) for k in keywords]
        if blinds is None:
            blinds = [1 + secrets.randbelow(P384_ORDER - 1) for _ in keywords]
        blinds = [int(r) for r in blinds]
        if len(blinds) != len(keywords):
            raise PirError(f"{len(blinds)} blinds for {len(keywords)} keywords")
        if any(not 0 < r < P384_ORDER for r in blinds):
            raise PirError("invalid OPRF blind: not in [1, n - 1]")
        data, offsets = _concatenate(keywords)
        count = len(keywords)
        packed = np.frombuffer(b"".join(r.to_bytes(OPRF_KEY_BYTES, "big") for r in blinds) or b"\0", dtype=np.uint8)
        queries = np.zeros((max(count, 1), OPRF_ELEMENT_BYTES), dtype=np.uint8)
        status = np.ones(max(count, 1), dtype=np.uint8)
        _check(load_library().hecuda_oprf_blind(_ptr(data), _ptr(offsets), count, _ptr(packed), _ptr(queries),
                                                _ptr(status)))
        return [OprfQueryContext(k, r, queries[i].tobytes()) for i, (k, r) in enumerate(zip(keywords, blinds))]

    def parse(self, response: bytes, context: OprfQueryContext) -> ParsedOprfOutput:
        """parse(oprfResponse:with:) (:106-117): PirError when the response does not verify."""
        parsed = self.parseMany([response], [context])[0]
        if parsed is None:
            raise PirError("invalidOprfResponse: the server's proof does not verify")
        return parsed

    def parseMany(self, responses: Sequence[bytes], contexts: Sequence[OprfQueryContext]) -> List[Optional[ParsedOprfOutput]]:
        """One parsed output per response in one device call; None where a response is rejected, including a wrong
        length."""
        responses = [bytes(r) for r in responses]
        if len(responses) != len(contexts):
            raise PirError(f"{len(responses)} responses for {len(contexts)} query contexts")
        sized = [i for i, r in enumerate(responses) if len(r) == OPRF_RESPONSE_BYTES]
        count = len(sized)
        data, offsets = _concatenate([contexts[i].keyword for i in sized])
        blinds = np.frombuffer(b"".join(contexts[i].blind.to_bytes(OPRF_KEY_BYTES, "big") for i in sized) or b"\0",
                               dtype=np.uint8)
        queries = np.frombuffer(b"".join(bytes(contexts[i].query) for i in sized) or b"\0", dtype=np.uint8)
        packed = np.frombuffer(b"".join(responses[i] for i in sized) or b"\0", dtype=np.uint8)
        outputs = np.zeros((max(count, 1), OPRF_OUTPUT_BYTES), dtype=np.uint8)
        status = np.ones(max(count, 1), dtype=np.uint8)
        _check(load_library().hecuda_oprf_finalize(_ptr(self._publicKey), _ptr(data), _ptr(offsets), count, _ptr(blinds),
                                                   _ptr(queries), _ptr(packed), _ptr(outputs), _ptr(status)))
        out: List[Optional[ParsedOprfOutput]] = [None] * len(responses)
        for j, i in enumerate(sized):
            if status[j] == 0:
                out[i] = ParsedOprfOutput.fromOprfOutput(outputs[j].tobytes(), self.configType)
        return out

    def decrypt(self, encryptedEntry: bytes, parsed: ParsedOprfOutput) -> bytes:
        """decrypt(encryptedEntry:with:) (:119-132): PirError when the entry does not authenticate."""
        value = self.decryptMany([encryptedEntry], [parsed])[0]
        if value is None:
            raise PirError("authenticationFailure: the entry does not open under its OPRF output")
        return value

    def decryptMany(self, encryptedEntries: Sequence[bytes], parsedOutputs: Sequence[ParsedOprfOutput]) -> List[Optional[bytes]]:
        """Every entry opened in one device call; None where an entry does not authenticate or is shorter than a tag."""
        entries = [bytes(e) for e in encryptedEntries]
        if len(entries) != len(parsedOutputs):
            raise PirError(f"{len(entries)} entries for {len(parsedOutputs)} parsed outputs")
        count = len(entries)
        sealed, offsets = _concatenate(entries)
        config = self.configType
        if any(len(p.nonce) != config.nonceSize or len(p.secretKey) != config.entryEncryptionKeySize
               for p in parsedOutputs):
            raise PirError("a parsed OPRF output has the wrong nonce or key size")
        # the device reads the nonce at h[0:12] and the key at h[24:48] of each OPRF output h
        outputs = np.frombuffer(b"".join(p.nonce + bytes(12) + p.secretKey for p in parsedOutputs) or b"\0",
                                dtype=np.uint8)
        values = np.zeros(max(int(offsets[-1]), 1), dtype=np.uint8)
        status = np.ones(max(count, 1), dtype=np.uint8)
        _check(load_library().hecuda_symmetric_pir_open(_ptr(outputs), _ptr(sealed), _ptr(offsets), count, _ptr(values),
                                                        _ptr(status)))
        tag = config.tagSize
        raw = values.tobytes()
        return [raw[int(offsets[i]):int(offsets[i + 1]) - tag] if status[i] == 0 else None for i in range(count)]
