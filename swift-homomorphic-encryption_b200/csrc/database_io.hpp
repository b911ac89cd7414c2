// database_io.hpp -- the host half of saving and loading processed PIR databases in the reference's format
// (ProcessedDatabase.serialize / init(from:context:), IndexPirProtocol.swift:286-378):
//
//   version byte (1) | plaintextCount (UInt32, little-endian) | per plaintext: tag 0 (nil) or tag 1 + PolyRq.serialize()
//
// A plaintext's offset depends on every tag before it, so the tags are walked here, once, before anything is
// allocated.  The walk gives every plaintext's tag offset; the device kernels (codec.cu, PolyLayout) read and write
// plaintexts at those offsets, and the pipelines (pir.cu) stage whole plaintexts in chunks planned from them.
#pragma once
#include <cstdint>
#include <vector>

namespace hecuda {
namespace dbio {

constexpr unsigned kVersion = 1;         // ProcessedDatabase.serializationVersion
constexpr long long kHeaderBytes = 5;    // version + UInt32 plaintextCount
constexpr long long kMaxCount = 0xffffffffll;

struct TagWalk {
    enum Error { kOk, kVersion, kTag, kTruncated } error = kOk;
    long long count = 0;  // plaintextCount
    unsigned value = 0;   // the version or tag that was refused
    long long at = -1;    // the plaintext whose tag or rows run past the end or whose tag was refused (-1: the header)
};

// Checks the header and walks the tags of the `byte_count` bytes at `bytes`, plaintext_bytes bytes per non-nil
// plaintext.  On success tag[p] is plaintext p's tag offset, for p < count, and tag[count] is where the last plaintext
// ends; bytes after it are ignored, as the reference ignores them.
inline TagWalk walk_tags(const unsigned char *bytes, long long byte_count, long long plaintext_bytes, std::vector<long long> &tag) {
    TagWalk w;
    tag.clear();
    if (byte_count < 1) return w.error = TagWalk::kTruncated, w;
    if (bytes[0] != kVersion) return w.error = TagWalk::kVersion, w.value = bytes[0], w;
    if (byte_count < kHeaderBytes) return w.error = TagWalk::kTruncated, w;
    w.count = (long long)bytes[1] | (long long)bytes[2] << 8 | (long long)bytes[3] << 16 | (long long)bytes[4] << 24;
    if (w.count > byte_count - kHeaderBytes) return w.error = TagWalk::kTruncated, w;  // one byte per plaintext at least
    tag.resize((size_t)w.count + 1);
    long long at = kHeaderBytes;
    for (long long p = 0; p < w.count; ++p) {
        tag[(size_t)p] = at;
        if (at >= byte_count) return w.error = TagWalk::kTruncated, w.at = p, w;
        const unsigned t = bytes[at];
        if (t > 1) return w.error = TagWalk::kTag, w.value = t, w.at = p, w;
        at += 1 + (t ? plaintext_bytes : 0);
        if (at > byte_count) return w.error = TagWalk::kTruncated, w.at = p, w;
    }
    tag[(size_t)w.count] = at;
    return w;
}

// The tag offsets of a serialization of `count` plaintexts with these presence flags (null: all present), the same
// as walk_tags gives for its bytes: tag[count] is the serialization's size.
inline void tag_offsets(const unsigned char *present, long long count, long long plaintext_bytes, std::vector<long long> &tag) {
    tag.resize((size_t)count + 1);
    long long at = kHeaderBytes;
    for (long long p = 0; p < count; ++p) {
        tag[(size_t)p] = at;
        at += 1 + (!present || present[p] ? plaintext_bytes : 0);
    }
    tag[(size_t)count] = at;
}

// Plaintexts [first, first + count) of a stream, staged as bytes [tag[first], tag[first + count]).
struct Chunk {
    long long first, count;
};

// Plaintexts [first, last) in consecutive chunks of whole plaintexts of at most `budget` bytes each; a plaintext larger
// than the budget is a chunk of its own.
inline std::vector<Chunk> plan_chunks(const std::vector<long long> &tag, long long first, long long last, long long budget) {
    std::vector<Chunk> plan;
    while (first < last) {
        long long end = first + 1;
        while (end < last && tag[(size_t)end + 1] - tag[(size_t)first] <= budget) ++end;
        plan.push_back({first, end - first});
        first = end;
    }
    return plan;
}

}  // namespace dbio
}  // namespace hecuda
