// keyword_pir.cuh -- index maps of the keyword-PIR kernels (keyword_pir.cu).  Every function is __host__ __device__,
// so the placement's CPU replay (tests/emu/keyword_pir_emulate.cu) computes exactly what the kernels compute.
//
//   HashKeyword.hash / hashIndices / indexFromHash      KeywordPir/HashBucket.swift:221-269
//   HashBucket.serialize (HashBucketEntry.serialize)     KeywordPir/HashBucket.swift:89-103, 176-187
#pragma once
#include <cstdint>

#include "sha256.cuh"

namespace hecuda {
namespace kwpir {

constexpr int kMaxRetries = 10;          // HashKeyword.maxRetries
constexpr int kSlotHeaderBytes = 10;     // keyword hash (8) + value length (2)
constexpr long long kMaxValueSize = 65535;  // HashBucketEntry.maxValueSize
constexpr int kMaxSlotCount = 255;       // HashBucket.maxSlotCount

// HashKeyword.hash: first 8 bytes of SHA-256(keyword), little-endian
SHA_HD uint64_t keyword_hash(const unsigned char *keyword, long long length) { return sha256::first8(keyword, length); }

// HashKeyword.indexFromHash: first8LE(SHA-256(bigEndian(hash) || counter)) % bucketCount
SHA_HD long long index_from_hash(uint64_t hash, long long bucket_count, int counter) {
    return (long long)(sha256::first8_9(hash, (uint32_t)counter) % (uint64_t)bucket_count);
}

// HashKeyword.hashIndices: out[0..h) -- each candidate retried with counters 1..maxRetries while it repeats an earlier
// one (across all h, as the reference does although the tables are disjoint)
SHA_HD void hash_indices(uint64_t hash, long long bucket_count, int h, int64_t *out) {
    for (int i = 0; i < h; ++i) {
        int counter = 0;
        long long index = index_from_hash(hash, bucket_count, counter);
        for (;;) {
            bool seen = false;
            for (int j = 0; j < i; ++j) seen |= out[j] == index;
            if (!seen || counter >= kMaxRetries) break;
            index = index_from_hash(hash, bucket_count, ++counter);
        }
        out[i] = index;
    }
}

// Byte j (< kSlotHeaderBytes + length) of one serialized HashBucketEntry: the keyword hash and the value length,
// both little-endian, then the value.
SHA_HD unsigned slot_byte(uint64_t hash, const unsigned char *value, long long length, long long j) {
    if (j < 8) return (unsigned)((hash >> (8 * j)) & 0xff);
    if (j < kSlotHeaderBytes) return (unsigned)(((unsigned long long)length >> (8 * (j - 8))) & 0xff);
    return value[j - kSlotHeaderBytes];
}

SHA_HD long long slot_size(long long value_length) { return kSlotHeaderBytes + value_length; }

}  // namespace kwpir
}  // namespace hecuda
