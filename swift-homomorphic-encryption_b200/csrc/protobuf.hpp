// protobuf.hpp -- the protobuf wire format on the host: one walker and one writer for every message the library reads or
// writes (PNNS databases and configs, pnns_database_io.hpp; PIR requests, keys and responses, pir_proto.hpp).
//
// The walker reads a message's fields in place and refuses what the reference's SwiftProtobuf decoding would refuse,
// or what would make a message mean two things: groups (wire types 3 and 4), varints longer than 10 bytes, a length
// that runs past its message, a singular message field given twice, and a known field with the wrong wire type.
// Unknown fields are stepped over.  The writer gives SwiftProtobuf's bytes: fields in number order, proto3 zero
// scalars omitted, set messages written even when empty, repeated scalars packed.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/hecuda.h"

namespace hecuda {
namespace proto {

enum Wire { kVarint = 0, kFixed64 = 1, kLen = 2, kFixed32 = 5 };
struct Error {
    int32_t code = HECUDA_OK;
    std::string what;
    bool set(int32_t c, const std::string &w) {
        code = c;
        what = w;
        return false;
    }
    bool invalid(const std::string &w) { return set(HECUDA_ERR_INVALID_ARGUMENT, w); }
};

// ------------------------------------------------------------------------------------------------ reading

// the varint at `at` (advanced past it): false when it runs past `end` or is longer than 10 bytes
inline bool read_varint(const unsigned char *b, long long end, long long &at, uint64_t &v, Error &e, const char *where) {
    v = 0;
    for (int k = 0; k < 10; ++k) {
        if (at >= end) return e.invalid(std::string("truncated(") + where + ": a varint runs past the end)");
        const unsigned char byte = b[at++];
        v |= (uint64_t)(byte & 0x7f) << (7 * k);
        if (!(byte & 0x80)) return true;
    }
    return e.invalid(std::string("malformedProtobuf(") + where + ": a varint longer than 10 bytes)");
}

// One field of a message: its number, wire type, and either its scalar value or its payload [begin, end)
struct Field {
    uint32_t number = 0;
    int wire = 0;
    uint64_t value = 0;
    long long begin = 0, end = 0;
};

// The fields of the message [at, end) of `b`, one at a time.  Groups and invalid wire types are refused, as is a
// length that runs past the message.
struct Fields {
    const unsigned char *b;
    long long at, end;
    const char *message;
    bool next(Field &f, Error &e) {  // false at the end of the message (e untouched) or on a refusal (e set)
        if (at >= end) return false;
        uint64_t key = 0;
        if (!read_varint(b, end, at, key, e, message)) return false;
        f.number = (uint32_t)(key >> 3);
        f.wire = (int)(key & 7);
        if (f.number == 0 || key >> 32)
            return e.invalid(std::string("malformedProtobuf(") + message + ": field number " + std::to_string(key >> 3) + ")");
        switch (f.wire) {
        case kVarint:
            return read_varint(b, end, at, f.value, e, message);
        case kFixed64:
        case kFixed32: {
            const int bytes = f.wire == kFixed64 ? 8 : 4;
            if (end - at < bytes) return e.invalid(std::string("truncated(") + message + ": a fixed-size field runs past the end)");
            f.value = 0;
            for (int k = 0; k < bytes; ++k) f.value |= (uint64_t)b[at + k] << (8 * k);
            at += bytes;
            return true;
        }
        case kLen: {
            uint64_t len = 0;
            if (!read_varint(b, end, at, len, e, message)) return false;
            if (len > (uint64_t)(end - at))
                return e.invalid(std::string("truncated(") + message + ": field " + std::to_string(f.number) + " of " +
                                 std::to_string(len) + " bytes runs past the end)");
            f.begin = at;
            f.end = at + (long long)len;
            at = f.end;
            return true;
        }
        case 3:
        case 4:
            return e.invalid(std::string("malformedProtobuf(") + message + ": groups are not supported)");
        default:
            return e.invalid(std::string("malformedProtobuf(") + message + ": wire type " + std::to_string(f.wire) + ")");
        }
    }
};

inline bool expect_wire(const Field &f, int wire, const char *message, Error &e) {
    if (f.wire == wire) return true;
    return e.invalid(std::string("malformedProtobuf(") + message + " field " + std::to_string(f.number) + ": wire type " +
                     std::to_string(f.wire) + ", expected " + std::to_string(wire) + ")");
}

// a singular message field: refused when given a second time (protobuf would merge the two)
inline bool first_time(bool &seen, const Field &f, const char *message, Error &e) {
    if (!expect_wire(f, kLen, message, e)) return false;
    if (seen)
        return e.invalid(std::string("malformedProtobuf(") + message + " field " + std::to_string(f.number) +
                         ": a singular message given twice)");
    seen = true;
    return true;
}

// a repeated varint field, packed (one length-delimited run) or not (one varint per field); at most `cap` values
inline bool repeated_varints(const unsigned char *b, const Field &f, std::vector<uint64_t> &out, size_t cap, const char *what,
                             Error &e) {
    if (f.wire == kVarint) {
        out.push_back(f.value);
    } else if (f.wire == kLen) {
        for (long long at = f.begin; at < f.end;) {
            uint64_t v = 0;
            if (!read_varint(b, f.end, at, v, e, what)) return false;
            out.push_back(v);
            if (out.size() > cap) break;
        }
    } else {
        return expect_wire(f, kVarint, what, e);
    }
    if (out.size() > cap)
        return e.set(HECUDA_ERR_UNSUPPORTED, std::string(what) + ": more than " + std::to_string(cap) + " values");
    return true;
}

inline bool scalar(const Field &f, const char *message, uint64_t &v, Error &e) {
    if (!expect_wire(f, kVarint, message, e)) return false;
    v = f.value;
    return true;
}

// ------------------------------------------------------------------------------------------------ writing

using Bytes = std::vector<unsigned char>;

inline int varint_size(uint64_t v) {
    int n = 1;
    while (v >>= 7) ++n;
    return n;
}
inline void put_varint(Bytes &out, uint64_t v) {
    while (v >= 0x80) {
        out.push_back((unsigned char)(v | 0x80));
        v >>= 7;
    }
    out.push_back((unsigned char)v);
}
inline void put_key(Bytes &out, uint32_t number, int wire) { put_varint(out, (uint64_t)number << 3 | (uint64_t)wire); }
inline void put_scalar(Bytes &out, uint32_t number, uint64_t v) {  // proto3: a zero scalar is not written
    if (!v) return;
    put_key(out, number, kVarint);
    put_varint(out, v);
}
inline void put_message(Bytes &out, uint32_t number, const Bytes &body) {  // a set message is written even when empty
    put_key(out, number, kLen);
    put_varint(out, body.size());
    out.insert(out.end(), body.begin(), body.end());
}
template <typename T>
inline void put_packed(Bytes &out, uint32_t number, const T *v, long long count) {
    if (count <= 0) return;
    Bytes body;
    for (long long k = 0; k < count; ++k) put_varint(body, (uint64_t)v[k]);
    put_message(out, number, body);
}

}  // namespace proto
}  // namespace hecuda
