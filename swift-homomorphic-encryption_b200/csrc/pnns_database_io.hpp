// pnns_database_io.hpp -- the host half of saving and loading processed PNNS databases in the reference's protobuf
// format (apple.swift_homomorphic_encryption.pnns.v1.SerializedProcessedDatabase, ProcessedDatabase.swift:56-88,
// PnnsConversion.swift), and of its ServerConfig and ClientConfig messages:
//
//   SerializedProcessedDatabase  1 plaintext_matrices (repeated SerializedPlaintextMatrix)  2 entry_ids (packed uint64)
//                                3 entry_metadatas (repeated bytes)  4 server_config
//   SerializedPlaintextMatrix    1 num_rows  2 num_columns  3 plaintexts (repeated { 1 poly bytes })  4 packing
//   ServerConfig                 1 client_config  2 database_packing
//   ClientConfig                 1 encryption_parameters  2 scaling_factor  3 query_packing  4 vector_dimension
//                                5 galois_elements (packed)  6 distance_metric  7 extra_plaintext_moduli (packed)
//   MatrixPacking                oneof 1 dense_row {}  2 diagonal { 2 baby_step_giant_step { 1 dim 2 baby 3 giant } }
//                                3 dense_column {}
//   v1.EncryptionParameters      1 polynomial_degree  2 plaintext_modulus  3 coefficient_moduli (packed)
//                                4 error_std_dev  5 security_level  6 he_scheme
//
// The packings and the config follow the plaintexts in the file, so the framing is walked here once, before anything is
// checked or allocated; the walk reads no payload and records where every plaintext's `poly` lies.  The writer gives
// SwiftProtobuf's bytes (fields in number order, proto3 zero scalars omitted, set messages written even when empty,
// repeated scalars packed) for everything but the payloads, and the offset of every plaintext's framing, which the
// serialize kernels (codec.cu, PolyLayout) write beside its rows.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/hecuda.h"
#include "protobuf.hpp"

namespace hecuda {
namespace pnnsio {

using namespace proto;

enum Packing { kUnset = 0, kDenseRow = 1, kDiagonal = 2, kDenseColumn = 3 };

inline bool unrecognized(const char *type, uint64_t value, Error &e) {
    return e.invalid(std::string("unrecognizedEnumValue(enum: ") + type + ", value: " + std::to_string((int32_t)value) + ")");
}

// MatrixPacking [begin, end) -> type and its BabyStepGiantStep (vector dimension, baby step, giant step)
inline bool parse_packing(const unsigned char *b, long long begin, long long end, int32_t &type, uint32_t bsgs[3], Error &e) {
    type = kUnset;
    bsgs[0] = bsgs[1] = bsgs[2] = 0;
    Fields fs{b, begin, end, "MatrixPacking"};
    Field f;
    bool seen[4] = {false, false, false, false};
    while (fs.next(f, e)) {
        if (f.number < 1 || f.number > 3) continue;  // unknown
        if (!first_time(seen[f.number], f, "MatrixPacking", e)) return false;
        type = (int32_t)f.number;  // a oneof: the last member given wins
        bsgs[0] = bsgs[1] = bsgs[2] = 0;
        Fields inner{b, f.begin, f.end, "MatrixPacking member"};
        Field g;
        bool has_bsgs = false;
        while (inner.next(g, e)) {
            if (type != kDiagonal || g.number != 2) continue;
            if (!first_time(has_bsgs, g, "MatrixPackingDiagonal", e)) return false;
            Fields steps{b, g.begin, g.end, "BabyStepGiantStep"};
            Field s;
            while (steps.next(s, e)) {
                if (s.number < 1 || s.number > 3) continue;
                uint64_t v = 0;
                if (!scalar(s, "BabyStepGiantStep", v, e)) return false;
                bsgs[s.number - 1] = (uint32_t)v;
            }
            if (e.code) return false;
        }
        if (e.code) return false;
        if (type == kDiagonal && !has_bsgs) return e.invalid("unsetField(MatrixPacking.diagonal.babyStepGiantStep)");
    }
    if (e.code) return false;
    if (type == kUnset) return e.invalid("unsetOneof(MatrixPacking.matrixPackingType)");
    return true;
}

inline bool parse_encryption_parameters(const unsigned char *b, long long begin, long long end, hecuda_pnns_server_config &c,
                                        Error &e) {
    const char *m = "EncryptionParameters";
    Fields fs{b, begin, end, m};
    Field f;
    std::vector<uint64_t> moduli;
    uint64_t v = 0;
    while (fs.next(f, e)) {
        switch (f.number) {
        case 1:
            if (!scalar(f, m, c.poly_degree, e)) return false;
            break;
        case 2:
            if (!scalar(f, m, c.plaintext_modulus, e)) return false;
            break;
        case 3:
            if (!repeated_varints(b, f, moduli, HECUDA_PNNS_MAX_COEFFICIENT_MODULI, "EncryptionParameters.coefficientModuli", e))
                return false;
            break;
        case 4:
            if (!scalar(f, m, v, e)) return false;
            c.error_std_dev = (int32_t)v;
            break;
        case 5:
            if (!scalar(f, m, v, e)) return false;
            c.security_level = (int32_t)v;
            break;
        case 6:
            if (!scalar(f, m, v, e)) return false;
            c.he_scheme = (int32_t)v;
            break;
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    c.coefficient_moduli_count = (int32_t)moduli.size();
    for (size_t k = 0; k < moduli.size(); ++k) c.coefficient_moduli[k] = moduli[k];
    // ConversionHe.swift: ErrorStdDev / SecurityLevel / HeScheme .native() and validate(scheme:)
    if (c.error_std_dev != 0 && c.error_std_dev != 1) return unrecognized("ErrorStdDev", (uint64_t)c.error_std_dev, e);
    if (c.security_level != 0 && c.security_level != 1) return unrecognized("SecurityLevel", (uint64_t)c.security_level, e);
    if (c.he_scheme == 2) return e.invalid("invalidScheme: BGV");
    if (c.he_scheme != 0 && c.he_scheme != 1) return unrecognized("HeScheme", (uint64_t)c.he_scheme, e);
    return true;
}

// ClientConfig [begin, end) into the client fields of `c`
inline bool parse_client_config(const unsigned char *b, long long begin, long long end, hecuda_pnns_server_config &c,
                                Error &e) {
    const char *m = "ClientConfig";
    Fields fs{b, begin, end, m};
    Field f;
    bool has_params = false, has_query_packing = false;
    long long params_at = 0, params_end = 0, packing_at = 0, packing_end = 0;
    std::vector<uint64_t> galois, extra;
    uint64_t v = 0;
    while (fs.next(f, e)) {
        switch (f.number) {
        case 1:
            if (!first_time(has_params, f, m, e)) return false;
            params_at = f.begin, params_end = f.end;
            break;
        case 2:
            if (!scalar(f, m, c.scaling_factor, e)) return false;
            break;
        case 3:
            if (!first_time(has_query_packing, f, m, e)) return false;
            packing_at = f.begin, packing_end = f.end;
            break;
        case 4:
            if (!scalar(f, m, v, e)) return false;
            c.vector_dimension = (uint32_t)v;
            break;
        case 5:
            if (!repeated_varints(b, f, galois, HECUDA_PNNS_MAX_GALOIS_ELEMENTS, "ClientConfig.galoisElements", e)) return false;
            break;
        case 6:
            if (!scalar(f, m, v, e)) return false;
            c.distance_metric = (int32_t)v;
            break;
        case 7:
            if (!repeated_varints(b, f, extra, HECUDA_PNNS_MAX_EXTRA_PLAINTEXT_MODULI, "ClientConfig.extraPlaintextModuli", e))
                return false;
            break;
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    // PnnsConversion.swift: ClientConfig.native()
    if (!has_params) return e.invalid("unsetField(ClientConfig.encryptionParameters)");
    if (!parse_encryption_parameters(b, params_at, params_end, c, e)) return false;
    uint32_t steps[3];
    if (!parse_packing(b, packing_at, packing_end, c.query_packing, steps, e)) return false;
    c.query_vector_dimension = steps[0], c.query_baby_step = steps[1], c.query_giant_step = steps[2];
    c.galois_element_count = (int32_t)galois.size();
    for (size_t k = 0; k < galois.size(); ++k) c.galois_elements[k] = (uint32_t)galois[k];
    if (c.distance_metric != 0) return unrecognized("DistanceMetric", (uint64_t)c.distance_metric, e);
    c.extra_plaintext_moduli_count = (int32_t)extra.size();
    for (size_t k = 0; k < extra.size(); ++k) c.extra_plaintext_moduli[k] = extra[k];
    return true;
}

inline bool parse_server_config(const unsigned char *b, long long begin, long long end, hecuda_pnns_server_config &c,
                                Error &e) {
    const char *m = "ServerConfig";
    Fields fs{b, begin, end, m};
    Field f;
    bool has_client = false, has_packing = false;
    long long client_at = 0, client_end = 0, packing_at = 0, packing_end = 0;
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!first_time(has_client, f, m, e)) return false;
            client_at = f.begin, client_end = f.end;
        } else if (f.number == 2) {
            if (!first_time(has_packing, f, m, e)) return false;
            packing_at = f.begin, packing_end = f.end;
        }
    }
    if (e.code) return false;
    if (!has_client) return e.invalid("unsetField(ServerConfig.clientConfig)");
    if (!parse_client_config(b, client_at, client_end, c, e)) return false;
    uint32_t steps[3];
    if (!parse_packing(b, packing_at, packing_end, c.database_packing, steps, e)) return false;
    c.database_vector_dimension = steps[0], c.database_baby_step = steps[1], c.database_giant_step = steps[2];
    return true;
}

// What one walk of a SerializedProcessedDatabase finds
struct Matrix {
    long long rows = 0, cols = 0;
    int32_t packing = kUnset;
    uint32_t bsgs[3] = {0, 0, 0};
    std::vector<long long> poly_at, poly_bytes;  // per plaintext, in file order
};
struct Database {
    std::vector<Matrix> matrices;
    std::vector<uint64_t> entry_ids;
    std::vector<long long> metadata_at, metadata_bytes;
    hecuda_pnns_server_config config{};
};

inline bool walk_matrix(const unsigned char *b, long long begin, long long end, Matrix &mx, Error &e) {
    const char *m = "SerializedPlaintextMatrix";
    Fields fs{b, begin, end, m};
    Field f;
    bool has_packing = false;
    long long packing_at = 0, packing_end = 0;
    uint64_t v = 0;
    while (fs.next(f, e)) {
        switch (f.number) {
        case 1:
        case 2:
            if (!scalar(f, m, v, e)) return false;
            (f.number == 1 ? mx.rows : mx.cols) = (long long)(uint32_t)v;
            break;
        case 3: {
            if (!expect_wire(f, kLen, m, e)) return false;
            Fields pt{b, f.begin, f.end, "SerializedPlaintext"};
            Field g;
            long long at = f.begin, bytes = 0;  // a plaintext without `poly` is an empty one
            while (pt.next(g, e))
                if (g.number == 1) {
                    if (!expect_wire(g, kLen, "SerializedPlaintext", e)) return false;
                    at = g.begin, bytes = g.end - g.begin;  // bytes: the last one given wins
                }
            if (e.code) return false;
            mx.poly_at.push_back(at);
            mx.poly_bytes.push_back(bytes);
            break;
        }
        case 4:
            if (!first_time(has_packing, f, m, e)) return false;
            packing_at = f.begin, packing_end = f.end;
            break;
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    return parse_packing(b, packing_at, packing_end, mx.packing, mx.bsgs, e);
}

// Walks the framing of the `size` bytes at `b` once; on success `db` says where every plaintext lies
inline bool walk_database(const unsigned char *b, long long size, Database &db, Error &e) {
    const char *m = "SerializedProcessedDatabase";
    Fields fs{b, 0, size, m};
    Field f;
    bool has_config = false;
    long long config_at = 0, config_end = 0;
    while (fs.next(f, e)) {
        switch (f.number) {
        case 1:
            if (!expect_wire(f, kLen, m, e)) return false;
            db.matrices.emplace_back();
            if (!walk_matrix(b, f.begin, f.end, db.matrices.back(), e)) return false;
            break;
        case 2:
            if (!repeated_varints(b, f, db.entry_ids, (size_t)size, "SerializedProcessedDatabase.entryIds", e)) return false;
            break;
        case 3:
            if (!expect_wire(f, kLen, m, e)) return false;
            db.metadata_at.push_back(f.begin);
            db.metadata_bytes.push_back(f.end - f.begin);
            break;
        case 4:
            if (!first_time(has_config, f, m, e)) return false;
            config_at = f.begin, config_end = f.end;
            break;
        default:  // an unknown field: Fields::next has stepped over it
            break;
        }
    }
    if (e.code) return false;
    if (!has_config) return e.invalid("unsetField(SerializedProcessedDatabase.serverConfig)");
    return parse_server_config(b, config_at, config_end, db.config, e);
}

// ------------------------------------------------------------------------------------------------ writing

inline Bytes encode_packing(int32_t type, uint32_t dim, uint32_t baby, uint32_t giant) {
    Bytes member, packing;
    if (type == kDiagonal) {
        Bytes steps;
        put_scalar(steps, 1, dim);
        put_scalar(steps, 2, baby);
        put_scalar(steps, 3, giant);
        put_message(member, 2, steps);
    }
    if (type != kUnset) put_message(packing, (uint32_t)type, member);
    return packing;
}

inline Bytes encode_client_config(const hecuda_pnns_server_config &c) {
    Bytes params, out;
    put_scalar(params, 1, c.poly_degree);
    put_scalar(params, 2, c.plaintext_modulus);
    put_packed(params, 3, c.coefficient_moduli, c.coefficient_moduli_count);
    put_scalar(params, 4, (uint64_t)(int64_t)c.error_std_dev);
    put_scalar(params, 5, (uint64_t)(int64_t)c.security_level);
    put_scalar(params, 6, (uint64_t)(int64_t)c.he_scheme);
    put_message(out, 1, params);
    put_scalar(out, 2, c.scaling_factor);
    put_message(out, 3, encode_packing(c.query_packing, c.query_vector_dimension, c.query_baby_step, c.query_giant_step));
    put_scalar(out, 4, c.vector_dimension);
    put_packed(out, 5, c.galois_elements, c.galois_element_count);
    put_scalar(out, 6, (uint64_t)(int64_t)c.distance_metric);
    put_packed(out, 7, c.extra_plaintext_moduli, c.extra_plaintext_moduli_count);
    return out;
}

inline Bytes encode_server_config(const hecuda_pnns_server_config &c) {
    Bytes out;
    put_message(out, 1, encode_client_config(c));
    put_message(out, 2, encode_packing(c.database_packing, c.database_vector_dimension, c.database_baby_step,
                                       c.database_giant_step));
    return out;
}

// The checks a config passes before it is written: the counts fit the arrays, and the enumerations are ones the
// reference writes (so that the library never writes a message it would refuse)
inline bool check_config(const hecuda_pnns_server_config &c, bool server, Error &e) {
    if (c.coefficient_moduli_count < 0 || c.coefficient_moduli_count > HECUDA_PNNS_MAX_COEFFICIENT_MODULI ||
        c.extra_plaintext_moduli_count < 0 || c.extra_plaintext_moduli_count > HECUDA_PNNS_MAX_EXTRA_PLAINTEXT_MODULI ||
        c.galois_element_count < 0 || c.galois_element_count > HECUDA_PNNS_MAX_GALOIS_ELEMENTS)
        return e.set(HECUDA_ERR_UNSUPPORTED, "a config count exceeds its array");
    if (c.error_std_dev != 0 && c.error_std_dev != 1) return unrecognized("ErrorStdDev", (uint64_t)c.error_std_dev, e);
    if (c.security_level != 0 && c.security_level != 1) return unrecognized("SecurityLevel", (uint64_t)c.security_level, e);
    if (c.he_scheme != 1) return e.invalid("invalidScheme: only BFV is written");
    if (c.distance_metric != 0) return unrecognized("DistanceMetric", (uint64_t)c.distance_metric, e);
    if (c.query_packing < kDenseRow || c.query_packing > kDenseColumn) return e.invalid("unsetOneof(ClientConfig.queryPacking)");
    if (server && (c.database_packing < kDenseRow || c.database_packing > kDenseColumn))
        return e.invalid("unsetOneof(ServerConfig.databasePacking)");
    return true;
}

// The bytes of a serialized database around its plaintexts.  Matrix k's plaintext p has its framing `frame` at
// tag[p] and its rows right after it; tag[count] is where the matrix's plaintexts end.  `head` is written at
// `head_at` (the matrix's field key and length, num_rows and num_columns) and `tail` right after tag[count] (its
// packing).  After the last matrix, `rest` (entry identifiers, metadata and the config) ends the file at `size`.
struct MatrixPlacement {
    long long head_at = 0;
    Bytes head, frame, tail;
    std::vector<long long> tag;
};
struct Placement {
    std::vector<MatrixPlacement> matrices;
    long long rest_at = 0, size = 0;
    Bytes rest;
};
struct MatrixShape {
    long long rows, cols, count, poly_bytes;
};

inline Placement place_database(const std::vector<MatrixShape> &shapes, const uint64_t *ids, long long id_count,
                                const unsigned char *metadata, const uint64_t *metadata_offsets, long long metadata_count,
                                const hecuda_pnns_server_config &c) {
    Placement pl;
    long long at = 0;
    for (const MatrixShape &s : shapes) {
        MatrixPlacement mp;
        Bytes fields;
        put_scalar(fields, 1, (uint64_t)s.rows);
        put_scalar(fields, 2, (uint64_t)s.cols);
        Bytes plaintext_head;  // SerializedPlaintext { 1 poly }
        put_key(plaintext_head, 1, kLen);
        put_varint(plaintext_head, (uint64_t)s.poly_bytes);
        put_key(mp.frame, 3, kLen);
        put_varint(mp.frame, (uint64_t)(plaintext_head.size() + s.poly_bytes));
        mp.frame.insert(mp.frame.end(), plaintext_head.begin(), plaintext_head.end());
        put_message(mp.tail, 4, encode_packing(c.database_packing, c.database_vector_dimension, c.database_baby_step,
                                               c.database_giant_step));
        const long long per = (long long)mp.frame.size() + s.poly_bytes;
        const long long body = (long long)fields.size() + s.count * per + (long long)mp.tail.size();
        mp.head_at = at;
        put_key(mp.head, 1, kLen);
        put_varint(mp.head, (uint64_t)body);
        mp.head.insert(mp.head.end(), fields.begin(), fields.end());
        at += (long long)mp.head.size();
        mp.tag.resize((size_t)s.count + 1);
        for (long long p = 0; p <= s.count; ++p) mp.tag[(size_t)p] = at + p * per;
        at += s.count * per + (long long)mp.tail.size();
        pl.matrices.push_back(std::move(mp));
    }
    put_packed(pl.rest, 2, ids, id_count);
    for (long long k = 0; k < metadata_count; ++k) {
        const uint64_t from = metadata_offsets[k], to = metadata_offsets[k + 1];
        put_key(pl.rest, 3, kLen);
        put_varint(pl.rest, to - from);
        pl.rest.insert(pl.rest.end(), metadata + from, metadata + to);
    }
    put_message(pl.rest, 4, encode_server_config(c));
    pl.rest_at = at;
    pl.size = at + (long long)pl.rest.size();
    return pl;
}

}  // namespace pnnsio
}  // namespace hecuda
