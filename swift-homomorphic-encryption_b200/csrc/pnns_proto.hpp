// pnns_proto.hpp -- the host half of answering PNNS requests in the reference's protobuf messages: the walk of what a
// client sends, and the framing of what it gets back.
//
//   pnns.v1.SerializedCiphertextMatrix  1 num_rows  2 num_columns  3 ciphertexts (repeated v1.SerializedCiphertext)
//                                       4 packing                  (pnns/v1/pnns.proto, SerializedCiphertextMatrix.swift)
//   pnns.v1.MatrixPacking               oneof 1 dense_row {}  2 diagonal {..}  3 dense_column {}
//                                                                  (pnns/v1/pnns_matrix_packing.proto)
//   api.pnns.v1.PNNSRequest             1 shard_indices (repeated uint32)  2 query (repeated SerializedCiphertextMatrix,
//                                       one per plaintext modulus)  3 evaluation_key_metadata { 1 timestamp  2 identifier }
//                                       4 config_id  5 evaluation_key { 1 metadata  2 evaluation_key }  6 shard_ids
//   api.pnns.v1.PNNSShardResponse       1 reply (repeated SerializedCiphertextMatrix)  2 entry_ids (packed uint64)
//                                       3 entry_metadatas (repeated bytes)          (api/pnns/v1/pnns.proto)
//
// A request's query is Query.proto() (PnnsConversion.swift:265-348): one `.denseRow` matrix of `.seeded` ciphertexts
// per plaintext modulus.  A response is Response.proto() (PnnsConversionApi.swift): one `.denseColumn` matrix per
// plaintext modulus of database rows x query rows, its ciphertexts serialized forDecryption (SerializedCiphertext.full
// with Bfv.skipLSBsForDecryption of that modulus' t and correction factor 1), then the database's entry ids and
// metadata.  The ciphertext walk is he_proto.hpp's, as for PIR.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "he_proto.hpp"
#include "protobuf.hpp"

namespace hecuda {
namespace pnnsproto {

using namespace proto;
using namespace heproto;

enum Packing { kUnset = 0, kDenseRow = 1, kDiagonal = 2, kDenseColumn = 3 };
inline const char *packing_name(int p) {
    return p == kDenseRow ? ".denseRow" : p == kDiagonal ? ".diagonal" : p == kDenseColumn ? ".denseColumn" : "unset";
}

// MatrixPacking [begin, end): which member of its oneof is set (the last one given wins)
inline bool walk_packing(const unsigned char *b, long long begin, long long end, int &packing, Error &e) {
    const char *m = "MatrixPacking";
    Fields fs{b, begin, end, m};
    Field f;
    bool seen[4] = {false, false, false, false};
    packing = kUnset;
    while (fs.next(f, e)) {
        if (f.number < 1 || f.number > 3) continue;
        if (!first_time(seen[f.number], f, m, e)) return false;
        packing = (int)f.number;
    }
    return e.code == HECUDA_OK;
}

// SerializedCiphertextMatrix [begin, end): its dimensions, packing and ciphertexts (each walked over `sz`; a null sz
// records the ciphertexts' ranges only)
struct Matrix {
    uint64_t rows = 0, columns = 0;
    int packing = kUnset;
    std::vector<Ciphertext> cts;
    std::vector<std::pair<long long, long long>> ranges;  // each ciphertext's [begin, end)
};
inline bool walk_matrix(const unsigned char *b, long long begin, long long end, const PolySizes *sz, Matrix &mx, Error &e) {
    const char *m = "SerializedCiphertextMatrix";
    Fields fs{b, begin, end, m};
    Field f;
    bool seen_packing = false;
    mx = Matrix{};
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!scalar(f, m, mx.rows, e)) return false;
        } else if (f.number == 2) {
            if (!scalar(f, m, mx.columns, e)) return false;
        } else if (f.number == 3) {
            if (!expect_wire(f, kLen, m, e)) return false;
            mx.ranges.emplace_back(f.begin, f.end);
            mx.cts.emplace_back();
            if (sz && !walk_ciphertext(b, f.begin, f.end, *sz, false, mx.cts.back(), e)) return false;
        } else if (f.number == 4) {
            if (!first_time(seen_packing, f, m, e)) return false;
            if (!walk_packing(b, f.begin, f.end, mx.packing, e)) return false;
        }
    }
    mx.rows = (uint32_t)mx.rows, mx.columns = (uint32_t)mx.columns;  // uint32 fields: protobuf keeps the low 32 bits
    return e.code == HECUDA_OK;
}

// EvaluationKeyMetadata [at, to) into the fields' key timestamp and identifier
inline bool walk_key_metadata(const unsigned char *b, long long at, long long to, hecuda_pnns_request_fields &r, Error &e) {
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
}

// PNNSRequest [0, size): every field.  query: each query matrix's [begin, end); shard_indices in message order;
// shard_ids: each id's [begin, end).  The fields' query_count and query_row_count come from the matrices' num_rows
// (refused when they differ).
struct Request {
    hecuda_pnns_request_fields fields{};
    std::vector<std::pair<long long, long long>> query, shard_ids;
    std::vector<uint64_t> shard_indices;
};
inline bool walk_pnns_request(const unsigned char *b, long long size, Request &r, Error &e) {
    const char *m = "PNNSRequest";
    r = Request{};
    hecuda_pnns_request_fields &x = r.fields;
    Fields fs{b, 0, size, m};
    Field f;
    bool seen_md = false, seen_key = false;
    long long key_metadata_at = -1, key_metadata_to = -1;
    while (fs.next(f, e)) {
        switch (f.number) {
        case 1:
            if (!repeated_varints(b, f, r.shard_indices, (size_t)1 << 32, "PNNSRequest.shardIndices", e)) return false;
            break;
        case 2: {
            if (!expect_wire(f, kLen, m, e)) return false;
            Matrix mx;
            if (!walk_matrix(b, f.begin, f.end, nullptr, mx, e)) return false;
            if (!r.query.empty() && mx.rows != (uint64_t)x.query_row_count)
                return e.invalid("invalidMatrixDimensions: query matrices of " + std::to_string(x.query_row_count) + " and " +
                                 std::to_string(mx.rows) + " rows");
            x.query_row_count = (uint32_t)mx.rows;
            r.query.emplace_back(f.begin, f.end);
            break;
        }
        case 3:
            if (!first_time(seen_md, f, m, e)) return false;
            if (!walk_key_metadata(b, f.begin, f.end, x, e)) return false;
            break;
        case 4:
            if (!expect_wire(f, kLen, m, e)) return false;
            x.config_id_offset = (uint64_t)f.begin, x.config_id_bytes = (uint64_t)(f.end - f.begin);
            break;
        case 5: {
            if (!first_time(seen_key, f, m, e)) return false;
            Fields ek{b, f.begin, f.end, "EvaluationKey"};
            Field g;
            bool seen_inner_md = false, seen_inner_key = false;
            x.has_evaluation_key = 1;
            while (ek.next(g, e)) {
                if (g.number == 1) {
                    if (!first_time(seen_inner_md, g, "EvaluationKey", e)) return false;
                    key_metadata_at = g.begin, key_metadata_to = g.end;
                } else if (g.number == 2) {
                    if (!first_time(seen_inner_key, g, "EvaluationKey", e)) return false;
                    x.evaluation_key_offset = (uint64_t)g.begin, x.evaluation_key_bytes = (uint64_t)(g.end - g.begin);
                }
            }
            if (e.code) return false;
            break;
        }
        case 6:
            if (!expect_wire(f, kLen, m, e)) return false;
            r.shard_ids.emplace_back(f.begin, f.end);
            break;
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    // the key's metadata: evaluation_key_metadata, or the metadata inside evaluation_key when that is absent
    if (!x.has_key_metadata && key_metadata_at >= 0 && !walk_key_metadata(b, key_metadata_at, key_metadata_to, x, e)) return false;
    x.query_count = (int32_t)r.query.size();
    x.shard_index_count = (int64_t)r.shard_indices.size();
    x.shard_id_count = (int64_t)r.shard_ids.size();
    return true;
}

// A request's query against the server: one .denseRow matrix per context, each of `columns` columns (the database's)
// and of the same rows, holding CiphertextMatrix.ciphertextCount(N, dims) ciphertexts, each over the context's
// sizes[k] (PnnsError's names; Server.computeResponse, PnnsConversion.swift)
inline bool walk_query(const unsigned char *b, const Request &r, const std::vector<PolySizes> &sizes, uint64_t columns,
                       std::vector<Matrix> &q, Error &e) {
    if (r.query.size() != sizes.size())
        return e.invalid("wrongCiphertextMatrixCount(got: " + std::to_string(r.query.size()) + ", expected: " +
                         std::to_string(sizes.size()) + ")");
    q.assign(r.query.size(), Matrix{});
    for (size_t k = 0; k < r.query.size(); ++k) {
        Matrix &mx = q[k];
        if (!walk_matrix(b, r.query[k].first, r.query[k].second, nullptr, mx, e)) return false;
        const long long n = sizes[k].n;
        if (mx.packing == kUnset) return e.invalid("unsetOneof(MatrixPacking.matrixPackingType)");
        if (mx.packing != kDenseRow)
            return e.invalid(std::string("wrongMatrixPacking(got: ") + packing_name(mx.packing) + ", expected: .denseRow)");
        if (mx.rows == 0 || mx.columns == 0 || mx.columns != columns || (long long)mx.columns > n / 2)
            return e.invalid("invalidMatrixDimensions(rowCount: " + std::to_string(mx.rows) + ", columnCount: " +
                             std::to_string(mx.columns) + ")");
        const long long per = 2 * ((n / 2) / [&] {
            long long p = 1;
            while (p < (long long)mx.columns) p <<= 1;
            return p;
        }());
        const long long expected = ((long long)mx.rows + per - 1) / per;
        if ((long long)mx.cts.size() != expected)
            return e.invalid("wrongCiphertextCount(got: " + std::to_string(mx.cts.size()) + ", expected: " +
                             std::to_string(expected) + ")");
        for (size_t i = 0; i < mx.ranges.size(); ++i)
            if (!walk_ciphertext(b, mx.ranges[i].first, mx.ranges[i].second, sizes[k], false, mx.cts[i], e)) return false;
    }
    return true;
}

// Bfv.skipLSBsForDecryption of a single-modulus ciphertext (Bfv+Decrypt.swift:51-110) over q0 with plaintext modulus t
inline void skip_lsbs_for_decryption(uint64_t q0, uint64_t t, long long n, int skip[2]) {
    auto bit_length = [](uint64_t v) {
        int b = 0;
        while (v) ++b, v >>= 1;
        return b;
    };
    const long long l_prime = q0 >= 2 * t ? bit_length(q0 / t) - 1 - 3 : 0;
    const long long spread = (long long)(8.0 * std::pow(2.0 * (double)n / 9.0, 0.5));
    const long long ceil_log2 = spread > 1 ? bit_length((uint64_t)spread - 1) : 0;
    long long p0 = std::max<long long>(l_prime, 0), p1 = l_prime - ceil_log2;
    if (p1 <= 1) p0 = std::max<long long>(l_prime + 1, 0), p1 = 0;
    skip[0] = (int)p0, skip[1] = (int)p1;
}

// ------------------------------------------------------------------------------------------------ writing

// One client's PNNSShardResponse: per context k a matrix of `replies` .full ciphertexts whose poly p has bytes[p]
// bytes (skip bits skip[p]), then the entry ids and metadata, the same for every client.  Everything but the reply
// polys is framing: frame() gives it as runs (offset, bytes).
struct ShardLayout {
    struct Part {
        long long bytes[2] = {0, 0}, at = 0, record = 0;  // at: the matrix field's offset
        int skip[2] = {0, 0};
        Bytes head, ct_head, ct_tail, packing;  // head: the matrix's key, length and dimensions
    };
    long long replies = 0, tail_at = 0, size = 0;
    std::vector<Part> parts;
    Bytes tail;
    long long poly_at(size_t k, long long r, int p) const {
        const Part &m = parts[k];
        return m.at + (long long)m.head.size() + r * m.record + (long long)m.ct_head.size() + (p ? m.bytes[0] : 0);
    }
    template <class F>
    void frame(F &&put) const {
        for (size_t k = 0; k < parts.size(); ++k) {
            const Part &m = parts[k];
            put(m.at, m.head);
            for (long long r = 0; r < replies; ++r) {
                const long long at = poly_at(k, r, 0);
                put(at - (long long)m.ct_head.size(), m.ct_head);
                put(at + m.bytes[0] + m.bytes[1], m.ct_tail);
            }
            put(m.at + (long long)m.head.size() + replies * m.record, m.packing);
        }
        put(tail_at, tail);
    }
};

// SerializedCiphertext { 2 full { 1 polys  2 skip_lsbs  3 correction_factor = 1 } } around polys of b0 + b1 bytes, as
// a repeated field `number`: (bytes before the polys, bytes after them)
inline void full_ciphertext_frame(uint32_t number, long long b0, long long b1, int skip0, int skip1, Bytes &head, Bytes &tail) {
    const long long polys = 2 + b0 + b1;  // Serialize.serializePolys: UInt16 count, then the polys
    const uint32_t skips[2] = {(uint32_t)skip0, (uint32_t)skip1};
    tail.clear();
    put_packed(tail, 2, skips, 2);
    put_scalar(tail, 3, 1);
    const long long full = 1 + varint_size((uint64_t)polys) + polys + (long long)tail.size();
    const long long ct = 1 + varint_size((uint64_t)full) + full;
    head.clear();
    put_key(head, number, kLen);
    put_varint(head, (uint64_t)ct);
    put_key(head, 2, kLen);  // SerializedCiphertext.full
    put_varint(head, (uint64_t)full);
    put_key(head, 1, kLen);  // SerializedFullCiphertext.polys
    put_varint(head, (uint64_t)polys);
    head.push_back(2);  // two polynomials
    head.push_back(0);
}

// bytes[k][p], skip[k][p]: context k's reply poly sizes and skip bits; rows x columns: database rows x query rows
inline ShardLayout place_shard_response(const std::vector<std::array<long long, 2>> &bytes,
                                        const std::vector<std::array<int, 2>> &skip, long long replies, uint64_t rows,
                                        uint64_t columns, const uint64_t *ids, long long id_count,
                                        const unsigned char *metadata, const uint64_t *metadata_offsets,
                                        long long metadata_count) {
    ShardLayout sl;
    sl.replies = replies;
    long long at = 0;
    for (size_t k = 0; k < bytes.size(); ++k) {
        ShardLayout::Part m;
        m.bytes[0] = bytes[k][0], m.bytes[1] = bytes[k][1], m.skip[0] = skip[k][0], m.skip[1] = skip[k][1];
        full_ciphertext_frame(3, m.bytes[0], m.bytes[1], m.skip[0], m.skip[1], m.ct_head, m.ct_tail);
        m.record = (long long)m.ct_head.size() + m.bytes[0] + m.bytes[1] + (long long)m.ct_tail.size();
        put_key(m.packing, 4, kLen);  // MatrixPacking { 3 dense_column {} }
        put_varint(m.packing, 2);
        put_key(m.packing, 3, kLen);
        put_varint(m.packing, 0);
        Bytes dims;
        put_scalar(dims, 1, rows);
        put_scalar(dims, 2, columns);
        const long long body = (long long)dims.size() + replies * m.record + (long long)m.packing.size();
        put_key(m.head, 1, kLen);  // PNNSShardResponse.reply
        put_varint(m.head, (uint64_t)body);
        m.head.insert(m.head.end(), dims.begin(), dims.end());
        m.at = at;
        at += (long long)m.head.size() + replies * m.record + (long long)m.packing.size();
        sl.parts.push_back(m);
    }
    put_packed(sl.tail, 2, ids, id_count);
    for (long long i = 0; i < metadata_count; ++i) {  // every element, even an empty one
        put_key(sl.tail, 3, kLen);
        put_varint(sl.tail, metadata_offsets[i + 1] - metadata_offsets[i]);
        sl.tail.insert(sl.tail.end(), metadata + metadata_offsets[i], metadata + metadata_offsets[i + 1]);
    }
    sl.tail_at = at;
    sl.size = at + (long long)sl.tail.size();
    return sl;
}

// What a client reads from a PNNSShardResponse: every matrix's dimensions, reply poly 0 offsets and skip bits; the ids
// decoded, and each metadata's [begin, end).  Refused unless every matrix is .denseColumn of the same dimensions and
// ciphertext count, its ciphertexts .full over the one-row sizes sizes[k] with one pair of skip bits.
struct ShardResponse {
    uint64_t rows = 0, columns = 0;
    long long replies = 0;
    std::vector<std::vector<long long>> poly_at;  // [matrix][reply]
    std::vector<std::array<int, 2>> skip;
    std::vector<uint64_t> ids;
    std::vector<std::pair<long long, long long>> metadata;
};
inline bool walk_shard_response(const unsigned char *b, long long size, const std::vector<PolySizes> &sizes, ShardResponse &r,
                                Error &e) {
    const char *m = "PNNSShardResponse";
    r = ShardResponse{};
    Fields fs{b, 0, size, m};
    Field f;
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!expect_wire(f, kLen, m, e)) return false;
            const size_t k = r.poly_at.size();
            if (k >= sizes.size())
                return e.invalid("wrongCiphertextMatrixCount(got: more than " + std::to_string(sizes.size()) + ")");
            Matrix mx;
            if (!walk_matrix(b, f.begin, f.end, &sizes[k], mx, e)) return false;
            if (mx.packing != kDenseColumn)
                return e.invalid(std::string("wrongMatrixPacking(got: ") + packing_name(mx.packing) + ", expected: .denseColumn)");
            if (k == 0) r.rows = mx.rows, r.columns = mx.columns, r.replies = (long long)mx.cts.size();
            if (mx.rows != r.rows || mx.columns != r.columns || (long long)mx.cts.size() != r.replies)
                return e.invalid("invalidResponse: reply matrices of different shapes");
            std::vector<long long> at;
            std::array<int, 2> skip{0, 0};
            for (size_t i = 0; i < mx.cts.size(); ++i) {
                const Ciphertext &ct = mx.cts[i];
                if (!ct.full) return e.invalid("invalidResponse: a reply ciphertext that is not .full");
                if (i == 0) skip = {ct.skip[0], ct.skip[1]};
                if (ct.skip[0] != skip[0] || ct.skip[1] != skip[1])
                    return e.invalid("invalidResponse: reply ciphertexts of one matrix with different skipLsbs");
                at.push_back(ct.poly[0]);
            }
            r.poly_at.push_back(at);
            r.skip.push_back(skip);
        } else if (f.number == 2) {
            if (!repeated_varints(b, f, r.ids, (size_t)1 << 40, "PNNSShardResponse.entryIds", e)) return false;
        } else if (f.number == 3) {
            if (!expect_wire(f, kLen, m, e)) return false;
            r.metadata.emplace_back(f.begin, f.end);
        }
    }
    if (e.code) return false;
    if (r.poly_at.size() != sizes.size())
        return e.invalid("wrongCiphertextMatrixCount(got: " + std::to_string(r.poly_at.size()) + ", expected: " +
                         std::to_string(sizes.size()) + ")");
    return true;
}

// SerializedCiphertextMatrix of `count` .seeded ciphertexts in .denseRow packing (SerializedCiphertextMatrix.proto())
inline Bytes encode_query_matrix(uint64_t rows, uint64_t columns, const unsigned char *poly0, const unsigned char *seeds,
                                 long long count, long long poly_bytes) {
    Bytes out;
    put_scalar(out, 1, rows);
    put_scalar(out, 2, columns);
    for (long long i = 0; i < count; ++i) {
        Bytes seeded, ct;
        put_key(seeded, 1, kLen);
        put_varint(seeded, (uint64_t)poly_bytes);
        seeded.insert(seeded.end(), poly0 + i * poly_bytes, poly0 + (i + 1) * poly_bytes);
        put_key(seeded, 2, kLen);
        put_varint(seeded, 32);
        seeded.insert(seeded.end(), seeds + 32 * i, seeds + 32 * (i + 1));
        put_message(ct, 1, seeded);
        put_message(out, 3, ct);
    }
    Bytes packing, dense_row;
    put_message(packing, 1, dense_row);
    put_message(out, 4, packing);
    return out;
}

}  // namespace pnnsproto
}  // namespace hecuda
