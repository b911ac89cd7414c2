// pir_proto.hpp -- the host half of answering PIR requests in the reference's protobuf messages: the walk of what a
// client sends, and the framing of what it gets back.
//
//   v1.SerializedCiphertext        the walk of he_proto.hpp (shared with the PNNS messages)
//   v1.SerializedCiphertextVec     1 ciphertexts (repeated)
//   v1.SerializedEvaluationKey     1 galois_key { 1 map<uint64, SerializedKeySwitchKey> }  2 relin_key { 1 relin_key }
//   v1.SerializedKeySwitchKey      1 key_switch_key (SerializedCiphertextVec)
//   pir.v1.EncryptedIndices        1 ciphertexts (repeated)  2 num_pir_calls            (PirConversion.swift:23-53)
//   api.pir.v1.PIRRequest          1 shard_index  2 query  3 evaluation_key_metadata { 1 timestamp  2 identifier }
//                                  4 configuration_hash  5 shard_id  6 evaluation_key { 1 metadata  2 evaluation_key }
//   api.pir.v1.PIRResponse         1 replies (repeated SerializedCiphertextVec)  2 stash  (PirConversionApi.swift:20-49)
//
// A walk reads no payload: it records where every ciphertext's polynomials and seed lie in the caller's bytes, so that
// the message crosses PCIe as it is and the device kernels read the payloads in place (PolyLayout tag / seed, drbg.cu).
// A reply is Response.proto(): SerializedCiphertext.full with Bfv.skipLSBsForDecryption and correction factor 1, the
// same framing for every reply of every client of one shape.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "he_proto.hpp"
#include "protobuf.hpp"

namespace hecuda {
namespace pirproto {

using namespace proto;
using namespace heproto;  // PolySizes, Ciphertext, walk_ciphertext

// EncryptedIndices [begin, end): its ciphertexts in order, and num_pir_calls (Query.indicesCount)
struct Query {
    std::vector<Ciphertext> cts;
    uint64_t indices = 0;
};
inline bool walk_encrypted_indices(const unsigned char *b, long long begin, long long end, const PolySizes &sz, Query &q,
                                   Error &e) {
    const char *m = "EncryptedIndices";
    Fields fs{b, begin, end, m};
    Field f;
    q = Query{};
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!expect_wire(f, kLen, m, e)) return false;
            q.cts.emplace_back();
            if (!walk_ciphertext(b, f.begin, f.end, sz, false, q.cts.back(), e)) return false;
        } else if (f.number == 2) {
            if (!scalar(f, m, q.indices, e)) return false;
        }
    }
    return e.code == HECUDA_OK;
}

// A walked query against the parameter's shape: num_pir_calls is the call's indices count, and the ciphertext count is
// the one the expansion takes (PirUtil.swift:326-327, as hecuda_mulpir_compute_response refuses it)
inline bool check_query(const Query &q, uint64_t indices, size_t ciphertexts, Error &e) {
    if (q.indices != indices)
        return e.invalid("invalidQuery: numPirCalls " + std::to_string(q.indices) + ", expected " + std::to_string(indices));
    if (q.cts.size() != ciphertexts)
        return e.invalid("expand: " + std::to_string(q.cts.size()) + " query ciphertexts, expected " + std::to_string(ciphertexts));
    return true;
}

// SerializedKeySwitchKey [begin, end): exactly `count` .seeded ciphertexts (one per coefficient modulus of the query)
inline bool walk_key_switch_key(const unsigned char *b, long long begin, long long end, const PolySizes &sz, int count,
                                std::vector<Ciphertext> &cts, Error &e) {
    Fields fs{b, begin, end, "SerializedKeySwitchKey"};
    Field f;
    bool seen = false;
    while (fs.next(f, e)) {
        if (f.number != 1) continue;
        if (!first_time(seen, f, "SerializedKeySwitchKey", e)) return false;
        Fields vec{b, f.begin, f.end, "SerializedCiphertextVec"};
        Field g;
        while (vec.next(g, e)) {
            if (g.number != 1) continue;
            if (!expect_wire(g, kLen, "SerializedCiphertextVec", e)) return false;
            cts.emplace_back();
            if (!walk_ciphertext(b, g.begin, g.end, sz, true, cts.back(), e)) return false;
        }
        if (e.code) return false;
        if ((int)cts.size() != count)
            return e.invalid("invalidKeySwitchingKey: " + std::to_string(cts.size()) + " ciphertexts, expected " +
                             std::to_string(count));
    }
    if (e.code) return false;
    if (!seen) return e.invalid("invalidKeySwitchingKey: 0 ciphertexts, expected " + std::to_string(count));
    return true;
}

// SerializedEvaluationKey [begin, end): the relinearization key if set, and the Galois keys in message order.
// ciphertexts: L key-switching ciphertexts per key, each over the L + 1 rows of `sz`.
struct GaloisKey {
    uint64_t element = 0;
    std::vector<Ciphertext> cts;
};
struct EvaluationKey {
    bool relin = false;
    std::vector<Ciphertext> relin_cts;
    std::vector<GaloisKey> galois;
    // every key ciphertext in message order: (key, ciphertext) with key -1 for the relinearization key
    std::vector<std::pair<int, int>> order;
};
inline bool walk_evaluation_key(const unsigned char *b, long long begin, long long end, const PolySizes &sz, int ciphertexts,
                                EvaluationKey &k, Error &e) {
    const char *m = "SerializedEvaluationKey";
    Fields fs{b, begin, end, m};
    Field f;
    bool has_galois = false, has_relin = false;
    k = EvaluationKey{};
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!first_time(has_galois, f, m, e)) return false;
            Fields map{b, f.begin, f.end, "SerializedGaloisKey"};
            Field entry;
            while (map.next(entry, e)) {
                if (entry.number != 1) continue;
                if (!expect_wire(entry, kLen, "SerializedGaloisKey", e)) return false;
                Fields kv{b, entry.begin, entry.end, "SerializedGaloisKey.KeySwitchKeysEntry"};
                Field g;
                uint64_t element = 0;  // a map entry's absent key is 0; its absent value an empty message
                bool has_value = false;
                long long at = entry.begin, to = entry.begin;
                while (kv.next(g, e)) {
                    if (g.number == 1) {
                        if (!scalar(g, "SerializedGaloisKey.KeySwitchKeysEntry", element, e)) return false;
                    } else if (g.number == 2) {
                        if (!first_time(has_value, g, "SerializedGaloisKey.KeySwitchKeysEntry", e)) return false;
                        at = g.begin, to = g.end;
                    }
                }
                if (e.code) return false;
                for (const GaloisKey &gk : k.galois)
                    if (gk.element == element) return e.invalid("repeated Galois element " + std::to_string(element));
                k.galois.push_back(GaloisKey{element, {}});
                if (!walk_key_switch_key(b, at, to, sz, ciphertexts, k.galois.back().cts, e)) return false;
                for (int i = 0; i < ciphertexts; ++i) k.order.emplace_back((int)k.galois.size() - 1, i);
            }
            if (e.code) return false;
        } else if (f.number == 2) {
            if (!first_time(has_relin, f, m, e)) return false;
            Fields rk{b, f.begin, f.end, "SerializedRelinKey"};
            Field g;
            bool seen = false;
            long long at = f.begin, to = f.begin;
            while (rk.next(g, e))
                if (g.number == 1) {
                    if (!first_time(seen, g, "SerializedRelinKey", e)) return false;
                    at = g.begin, to = g.end;
                }
            if (e.code) return false;
            k.relin = true;
            if (!walk_key_switch_key(b, at, to, sz, ciphertexts, k.relin_cts, e)) return false;
            for (int i = 0; i < ciphertexts; ++i) k.order.emplace_back(-1, i);
        }
    }
    return e.code == HECUDA_OK;
}

// PIRRequest [0, size): every field, with the byte ranges of the query, the key and the metadata's bytes
inline bool walk_pir_request(const unsigned char *b, long long size, hecuda_pir_request_fields &r, Error &e) {
    const char *m = "PIRRequest";
    r = hecuda_pir_request_fields{};
    Fields fs{b, 0, size, m};
    Field f;
    bool seen[7] = {false, false, false, false, false, false, false};
    auto metadata = [&](long long at, long long to) {
        Fields md{b, at, to, "EvaluationKeyMetadata"};
        Field g;
        while (md.next(g, e)) {
            if (g.number == 1) {
                if (!scalar(g, "EvaluationKeyMetadata", r.key_timestamp, e)) return false;
            } else if (g.number == 2) {
                if (!expect_wire(g, kLen, "EvaluationKeyMetadata", e)) return false;
                r.key_identifier_offset = (uint64_t)g.begin, r.key_identifier_bytes = (uint64_t)(g.end - g.begin);
            }
        }
        r.has_key_metadata = 1;
        return e.code == HECUDA_OK;
    };
    long long key_metadata_at = -1, key_metadata_to = -1;
    while (fs.next(f, e)) {
        uint64_t v = 0;
        switch (f.number) {
        case 1:
            if (!scalar(f, m, v, e)) return false;
            r.shard_index = (uint32_t)v;
            break;
        case 2:
            if (!first_time(seen[2], f, m, e)) return false;
            r.has_query = 1, r.query_offset = (uint64_t)f.begin, r.query_bytes = (uint64_t)(f.end - f.begin);
            break;
        case 3:
            if (!first_time(seen[3], f, m, e)) return false;
            if (!metadata(f.begin, f.end)) return false;
            break;
        case 4:
            if (!expect_wire(f, kLen, m, e)) return false;
            r.configuration_hash_offset = (uint64_t)f.begin, r.configuration_hash_bytes = (uint64_t)(f.end - f.begin);
            break;
        case 5:
            if (!expect_wire(f, kLen, m, e)) return false;
            r.has_shard_id = 1, r.shard_id_offset = (uint64_t)f.begin, r.shard_id_bytes = (uint64_t)(f.end - f.begin);
            break;
        case 6: {
            if (!first_time(seen[6], f, m, e)) return false;
            Fields ek{b, f.begin, f.end, "EvaluationKey"};
            Field g;
            bool seen_md = false, seen_key = false;
            r.has_evaluation_key = 1;
            while (ek.next(g, e)) {
                if (g.number == 1) {
                    if (!first_time(seen_md, g, "EvaluationKey", e)) return false;
                    key_metadata_at = g.begin, key_metadata_to = g.end;
                } else if (g.number == 2) {
                    if (!first_time(seen_key, g, "EvaluationKey", e)) return false;
                    r.evaluation_key_offset = (uint64_t)g.begin, r.evaluation_key_bytes = (uint64_t)(g.end - g.begin);
                }
            }
            if (e.code) return false;
            break;
        }
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    // the key's metadata: evaluation_key_metadata, or the metadata inside evaluation_key when that is absent
    if (!r.has_key_metadata && key_metadata_at >= 0 && !metadata(key_metadata_at, key_metadata_to)) return false;
    return true;
}

// ------------------------------------------------------------------------------------------------ writing

// One client's PIRResponse for `indices` replies of `chunks` ciphertexts each.  Reply ciphertext r (= index x chunks +
// chunk) has its poly 0 at poly_at(r, 0) and poly 1 right after it; the bytes around them are the same for every
// ciphertext: `vec_head` opens each reply (before its first ciphertext), `ct_head` precedes poly 0, `ct_tail` follows
// poly 1.
struct ResponseLayout {
    long long indices = 0, chunks = 0, bytes[2] = {0, 0};
    Bytes vec_head, ct_head, ct_tail;
    long long record = 0, reply = 0, size = 0;
    long long poly_at(long long r, int p) const {
        const long long index = r / chunks, chunk = r - index * chunks;
        return index * reply + (long long)vec_head.size() + chunk * record + (long long)ct_head.size() + (p ? bytes[0] : 0);
    }
    // the framing of ciphertext r: (offset, bytes) of each of its runs, in order
    template <class F>
    void frame(long long r, F &&put) const {
        const long long at = poly_at(r, 0);
        if (r % chunks == 0) put(at - (long long)ct_head.size() - (long long)vec_head.size(), vec_head);
        put(at - (long long)ct_head.size(), ct_head);
        put(at + bytes[0] + bytes[1], ct_tail);
    }
};

inline ResponseLayout place_response(long long indices, long long chunks, long long bytes0, long long bytes1, int skip0,
                                     int skip1) {
    ResponseLayout rl;
    rl.indices = indices, rl.chunks = chunks, rl.bytes[0] = bytes0, rl.bytes[1] = bytes1;
    const long long polys = 2 + bytes0 + bytes1;  // Serialize.serializePolys: UInt16 count, then the polys
    const uint32_t skips[2] = {(uint32_t)skip0, (uint32_t)skip1};
    Bytes tail;  // SerializedFullCiphertext fields 2 and 3
    put_packed(tail, 2, skips, 2);
    put_scalar(tail, 3, 1);
    const long long full = 1 + varint_size((uint64_t)polys) + polys + (long long)tail.size();
    const long long ct = 1 + varint_size((uint64_t)full) + full;  // SerializedCiphertext { 2 full }
    Bytes head;
    put_key(head, 1, kLen);  // SerializedCiphertextVec.ciphertexts
    put_varint(head, (uint64_t)ct);
    put_key(head, 2, kLen);  // SerializedCiphertext.full
    put_varint(head, (uint64_t)full);
    put_key(head, 1, kLen);  // SerializedFullCiphertext.polys
    put_varint(head, (uint64_t)polys);
    head.push_back(2);  // two polynomials
    head.push_back(0);
    rl.ct_head = head;
    rl.ct_tail = tail;
    rl.record = (long long)head.size() + bytes0 + bytes1 + (long long)tail.size();
    const long long vec = chunks * rl.record;
    put_key(rl.vec_head, 1, kLen);  // PIRResponse.replies
    put_varint(rl.vec_head, (uint64_t)vec);
    rl.reply = (long long)rl.vec_head.size() + vec;
    rl.size = indices * rl.reply;
    return rl;
}

// Where the reply ciphertexts of a PIRResponse lie: refused unless it holds `indices` replies of `chunks` .full
// ciphertexts of two polys each, packed with skip[0] / skip[1] low bits dropped over the one-row sizes `sz`
inline bool walk_pir_response(const unsigned char *b, long long size, const PolySizes &sz, long long indices,
                              long long chunks, int skip0, int skip1, std::vector<long long> &poly_at, Error &e) {
    Fields fs{b, 0, size, "PIRResponse"};
    Field f;
    long long replies = 0;
    poly_at.clear();
    while (fs.next(f, e)) {
        if (f.number != 1) continue;  // the stash (2) is not read
        if (!expect_wire(f, kLen, "PIRResponse", e)) return false;
        ++replies;
        Fields vec{b, f.begin, f.end, "SerializedCiphertextVec"};
        Field g;
        long long count = 0;
        while (vec.next(g, e)) {
            if (g.number != 1) continue;
            if (!expect_wire(g, kLen, "SerializedCiphertextVec", e)) return false;
            Ciphertext ct;
            if (!walk_ciphertext(b, g.begin, g.end, sz, false, ct, e)) return false;
            if (!ct.full || ct.skip[0] != skip0 || ct.skip[1] != skip1)
                    return e.invalid("invalidResponse: a reply ciphertext that is not .full with skipLsbs [" +
                                 std::to_string(skip0) + ", " + std::to_string(skip1) + "]");
            poly_at.push_back(ct.poly[0]);
            ++count;
        }
        if (e.code) return false;
        if (count != chunks)
            return e.invalid("invalidResponse: " + std::to_string(count) + " ciphertexts in a reply, expected " +
                             std::to_string(chunks));
    }
    if (e.code) return false;
    if (replies != indices)
        return e.invalid("invalidResponse: " + std::to_string(replies) + " replies, expected " + std::to_string(indices));
    return true;
}

// EncryptedIndices of `count` .seeded ciphertexts (poly0: count x poly_bytes, seeds: count x 32), as Query.proto()
inline Bytes encode_encrypted_indices(const unsigned char *poly0, const unsigned char *seeds, long long count,
                                      long long poly_bytes, uint64_t indices) {
    Bytes out;
    for (long long i = 0; i < count; ++i) {
        Bytes seeded, ct;
        put_key(seeded, 1, kLen);
        put_varint(seeded, (uint64_t)poly_bytes);
        seeded.insert(seeded.end(), poly0 + i * poly_bytes, poly0 + (i + 1) * poly_bytes);
        put_key(seeded, 2, kLen);
        put_varint(seeded, 32);
        seeded.insert(seeded.end(), seeds + 32 * i, seeds + 32 * (i + 1));
        put_message(ct, 1, seeded);
        put_message(out, 1, ct);
    }
    put_scalar(out, 2, indices);
    return out;
}

// SerializedKeySwitchKey of `count` .seeded ciphertexts
inline Bytes encode_key_switch_key(const unsigned char *poly0, const unsigned char *seeds, long long count,
                                   long long poly_bytes) {
    Bytes vec, key;
    for (long long i = 0; i < count; ++i) {
        Bytes seeded, ct;
        put_key(seeded, 1, kLen);
        put_varint(seeded, (uint64_t)poly_bytes);
        seeded.insert(seeded.end(), poly0 + i * poly_bytes, poly0 + (i + 1) * poly_bytes);
        put_key(seeded, 2, kLen);
        put_varint(seeded, 32);
        seeded.insert(seeded.end(), seeds + 32 * i, seeds + 32 * (i + 1));
        put_message(ct, 1, seeded);
        put_message(vec, 1, ct);
    }
    put_message(key, 1, vec);
    return key;
}

}  // namespace pirproto
}  // namespace hecuda
