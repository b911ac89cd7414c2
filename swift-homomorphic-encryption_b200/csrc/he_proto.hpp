// he_proto.hpp -- v1.SerializedCiphertext on the host, shared by every server that reads the reference's protobuf
// messages (PIR requests, pir_proto.hpp; PNNS requests, pnns_proto.hpp):
//
//   v1.SerializedCiphertext        oneof 1 seeded { 1 poly0  2 seed }  2 full { 1 polys  2 skip_lsbs (packed)
//                                  3 correction_factor }                       (he.proto, ConversionHe.swift:90-135)
//
// A walk reads no payload: it records where the ciphertext's polynomials and seed lie in the caller's bytes.  `.full`
// polys are Serialize.serializePolys' bytes (Serialize.swift:29-69): a little-endian UInt16 polynomial count, then each
// polynomial packed with its skip_lsbs.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "protobuf.hpp"

namespace hecuda {
namespace heproto {

using namespace proto;

// The serialized size of one polynomial over rows of `bits` bits each at degree n: sum over rows of ceil(n (bits - skip) /
// 8) (PolyContext.serializationByteCount); -1 when skip is not below every row's bit count (invalidCoefficientPacking)
struct PolySizes {
    long long n = 0;
    std::vector<int> bits;
    long long bytes(long long skip) const {
        long long total = 0;
        for (int b : bits) {
            if (skip < 0 || skip >= b) return -1;
            total += (n * (b - skip) + 7) / 8;
        }
        return total;
    }
};

// the sizes of a codec's rows (CodecConsts of kernels.cuh: rows, width[] at skipLSBs 0)
template <class Codec>
inline PolySizes poly_sizes(const Codec &cc, long long n) {
    PolySizes sz;
    sz.n = n;
    sz.bits.assign(cc.width, cc.width + cc.rows);
    return sz;
}

// Where one ciphertext lies in a message.  poly[p]: offset of polynomial p's bytes (a seeded ciphertext has poly[0] only);
// seed: offset of its 32-byte seed (seeded only); skip[p]: the low bits polynomial p omits (.full only)
struct Ciphertext {
    bool full = false;
    long long poly[2] = {0, 0}, seed = -1;
    int skip[2] = {0, 0};
};

// SerializedCiphertext [begin, end) as SerializedCiphertext.native() and Ciphertext(deserialize:) read it: poly0 (and a
// .full ciphertext's two polys) of the serialized size over `sz`, a 32-byte seed, a correction factor of 1.  key: an
// evaluation-key ciphertext, which must be .seeded (the form key generation writes).
inline bool walk_ciphertext(const unsigned char *b, long long begin, long long end, const PolySizes &sz, bool key,
                            Ciphertext &ct, Error &e) {
    const char *m = "SerializedCiphertext";
    Fields fs{b, begin, end, m};
    Field f;
    bool seen[3] = {false, false, false};
    int type = 0;
    long long at = 0, to = 0;
    while (fs.next(f, e)) {
        if (f.number != 1 && f.number != 2) continue;  // unknown
        if (!first_time(seen[f.number], f, m, e)) return false;
        type = (int)f.number;  // a oneof: the last member given wins
        at = f.begin, to = f.end;
    }
    if (e.code) return false;
    if (type == 0) return e.invalid("unsetOneof(SerializedCiphertext.serializedCiphertextType)");
    ct = Ciphertext{};
    if (type == 1) {  // SerializedSeededCiphertext
        Fields inner{b, at, to, "SerializedSeededCiphertext"};
        long long poly_at = at, poly_bytes = 0, seed_at = at, seed_bytes = 0;  // proto3 bytes: absent is empty
        while (inner.next(f, e)) {
            if (f.number != 1 && f.number != 2) continue;
            if (!expect_wire(f, kLen, "SerializedSeededCiphertext", e)) return false;
            (f.number == 1 ? poly_at : seed_at) = f.begin;  // the last one given wins
            (f.number == 1 ? poly_bytes : seed_bytes) = f.end - f.begin;
        }
        if (e.code) return false;
        if (poly_bytes != sz.bytes(0))
            return e.invalid("serializedBufferSizeMismatch(poly0: " + std::to_string(poly_bytes) + " bytes, expected " +
                             std::to_string(sz.bytes(0)) + ")");
        if (seed_bytes != 32) return e.invalid("invalid seed: " + std::to_string(seed_bytes) + " bytes, expected 32");
        ct.poly[0] = poly_at;
        ct.seed = seed_at;
        return true;
    }
    if (key) return e.set(HECUDA_ERR_UNSUPPORTED, "SerializedCiphertext.full evaluation-key ciphertexts are not supported");
    Fields inner{b, at, to, "SerializedFullCiphertext"};
    long long polys_at = at, polys_bytes = 0;
    uint64_t correction = 0;
    std::vector<uint64_t> skips;
    while (inner.next(f, e)) {
        if (f.number == 1) {
            if (!expect_wire(f, kLen, "SerializedFullCiphertext", e)) return false;
            polys_at = f.begin, polys_bytes = f.end - f.begin;
        } else if (f.number == 2) {
            if (!repeated_varints(b, f, skips, 2, "SerializedFullCiphertext.skipLsbs", e)) return false;
        } else if (f.number == 3) {
            if (!scalar(f, "SerializedFullCiphertext", correction, e)) return false;
        }
    }
    if (e.code) return false;
    if (correction != 1)
        return e.set(HECUDA_ERR_UNSUPPORTED, "SerializedCiphertext.full with correctionFactor " + std::to_string(correction) +
                                                 ": only 1 is supported");
    if (polys_bytes < 2) return e.invalid("serializationBufferSizeMismatch(polys: " + std::to_string(polys_bytes) + " bytes)");
    const unsigned polys = b[polys_at] | (unsigned)b[polys_at + 1] << 8;
    if (polys != 2) return e.invalid("invalidCiphertext: " + std::to_string(polys) + " polynomials, expected 2");
    if (!skips.empty() && skips.size() != 2)
        return e.invalid("invalidCiphertext: " + std::to_string(skips.size()) + " skipLsbs for 2 polynomials");
    long long expected = 2;
    for (int p = 0; p < 2; ++p) {
        const long long skip = skips.empty() ? 0 : (long long)std::min<uint64_t>(skips[p], 1u << 20);
        const long long bytes = sz.bytes(skip);
        if (bytes < 0) return e.invalid("invalidCoefficientPacking(skipLSBs: " + std::to_string(skip) + ")");
        ct.skip[p] = (int)skip;
        ct.poly[p] = polys_at + expected;
        expected += bytes;
    }
    if (polys_bytes != expected)
        return e.invalid("serializedBufferSizeMismatch(polys: " + std::to_string(polys_bytes) + " bytes, expected " +
                         std::to_string(expected) + ")");
    ct.full = true;
    return true;
}

}  // namespace heproto
}  // namespace hecuda
