// simple_pir_proto.hpp -- the host half of answering SimplePIR requests in the reference's protobuf messages, and of
// reading and writing the SimplePIRConfig the SimplePIRProcessDatabase tool writes beside its shards.
//
//   pir.v1.SimplePIRMatrix            1 row_count  2 col_count  3 data (repeated uint64, row-major)
//   api.pir.v1.SimplePIRRequest       1 request (SimplePIRMatrix)  2 shard_index  3 configuration_hash (bytes)
//   api.pir.v1.SimplePIRResponse      1 response (SimplePIRMatrix)
//   pir.v1.SimplePIREncryptionParams  1 lattice_dimension  2 error_std_dev (double)  3 plaintext_bits  4 ciphertext_bits
//   pir.v1.SimplePIRParameters        1 encryption_params  2 a_seed  3 entry_size_in_bytes  4 entries_per_column
//                                     5 chunks_per_entry  6 database_columns
//   pir.v1.DatabaseMapping            1 entries (repeated Entry { 1 original_index  2 size  3 chunks (repeated
//                                     ChunkLocation { 1 shard_index  2 index }) })  2 chunk_size
//   api.pir.v1.SimplePIRConfig        1 database_mapping  2 params (repeated)  3 hint_identifiers (repeated bytes)
//                                     (pir/v1/simple_pir.proto, api/pir/v1/pir.proto)
//
// Conversions: Array2d.proto() / SimplePIRMatrix.native() (PirConversion.swift:380-401), SimplePirEncryptionParams,
// SimplePirParameters and DatabaseMap (:403-518).  The request walk records where a matrix's `data` lies -- packed
// runs, or single unpacked elements, each as one byte run -- and never reads it: the device decodes it
// (simple_pir.cu).  Every uint32 field keeps the low 32 bits of its varint, as protobuf does.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "protobuf.hpp"

namespace hecuda {
namespace spirproto {

using namespace proto;

// SimplePIRMatrix [begin, end): its dimensions and the byte runs of its data, in message order.  An unpacked element
// is the run of its one varint (the field's value bytes, after its key).
struct Matrix {
    uint32_t rows = 0, columns = 0;
    std::vector<std::pair<long long, long long>> runs;
};
inline bool walk_matrix(const unsigned char *b, long long begin, long long end, Matrix &mx, Error &e) {
    const char *m = "SimplePIRMatrix";
    Fields fs{b, begin, end, m};
    Field f;
    mx = Matrix{};
    uint64_t v = 0;
    for (long long key_at = fs.at; fs.next(f, e); key_at = fs.at) {
        if (f.number == 1) {
            if (!scalar(f, m, v, e)) return false;
            mx.rows = (uint32_t)v;
        } else if (f.number == 2) {
            if (!scalar(f, m, v, e)) return false;
            mx.columns = (uint32_t)v;
        } else if (f.number == 3) {
            if (f.wire == kLen) {
                if (f.end > f.begin) mx.runs.emplace_back(f.begin, f.end);
            } else if (f.wire == kVarint) {
                uint64_t key = 0;
                read_varint(b, end, key_at, key, e, m);  // read once already: key_at is now the value's first byte
                mx.runs.emplace_back(key_at, fs.at);
            } else {
                return expect_wire(f, kVarint, m, e);
            }
        }
    }
    return e.code == HECUDA_OK;
}

// SimplePIRRequest [0, size)
struct Request {
    bool has_request = false;
    Matrix matrix;
    uint32_t shard_index = 0;
    long long hash_begin = 0, hash_end = 0;
};
inline bool walk_request(const unsigned char *b, long long size, Request &r, Error &e) {
    const char *m = "SimplePIRRequest";
    r = Request{};
    Fields fs{b, 0, size, m};
    Field f;
    uint64_t v = 0;
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!first_time(r.has_request, f, m, e)) return false;
            if (!walk_matrix(b, f.begin, f.end, r.matrix, e)) return false;
        } else if (f.number == 2) {
            if (!scalar(f, m, v, e)) return false;
            r.shard_index = (uint32_t)v;
        } else if (f.number == 3) {
            if (!expect_wire(f, kLen, m, e)) return false;
            r.hash_begin = f.begin, r.hash_end = f.end;
        }
    }
    return e.code == HECUDA_OK;
}

// SimplePIRResponse [0, size) with its data decoded (the client side; at most `cap` values)
struct Response {
    bool has_response = false;
    uint32_t rows = 0, columns = 0;
    std::vector<uint64_t> data;
};
inline bool walk_response(const unsigned char *b, long long size, size_t cap, Response &r, Error &e) {
    const char *m = "SimplePIRResponse";
    r = Response{};
    Fields fs{b, 0, size, m};
    Field f;
    while (fs.next(f, e)) {
        if (f.number != 1) continue;
        if (!first_time(r.has_response, f, m, e)) return false;
        Fields inner{b, f.begin, f.end, "SimplePIRMatrix"};
        Field g;
        uint64_t v = 0;
        while (inner.next(g, e)) {
            if (g.number == 1) {
                if (!scalar(g, "SimplePIRMatrix", v, e)) return false;
                r.rows = (uint32_t)v;
            } else if (g.number == 2) {
                if (!scalar(g, "SimplePIRMatrix", v, e)) return false;
                r.columns = (uint32_t)v;
            } else if (g.number == 3) {
                if (!repeated_varints(b, g, r.data, cap, "SimplePIRMatrix.data", e)) return false;
            }
        }
        if (e.code != HECUDA_OK) return false;
    }
    if (e.code != HECUDA_OK) return false;
    if (r.data.size() != (size_t)r.rows * r.columns)
        return e.invalid("SimplePIRMatrix: " + std::to_string(r.data.size()) + " values for " + std::to_string(r.rows) +
                         " x " + std::to_string(r.columns));
    return true;
}

// Array2d.proto() as a SimplePIRMatrix body
inline Bytes encode_matrix(uint32_t rows, uint32_t columns, const uint64_t *data, long long count) {
    Bytes body;
    put_scalar(body, 1, rows);
    put_scalar(body, 2, columns);
    put_packed(body, 3, data, count);
    return body;
}

// ------------------------------------------------------------------------------------------------ SimplePIRConfig

// one SimplePIRParameters: the library's params (word_bits from ct, as the tool chooses its Scalar) and the seed range
struct Params {
    hecuda_simple_pir_params p{};
    double error_std_dev = 0;
    long long seed_begin = 0, seed_end = 0;
};

inline bool walk_encryption_params(const unsigned char *b, long long begin, long long end, Params &x, Error &e) {
    const char *m = "SimplePIREncryptionParams";
    Fields fs{b, begin, end, m};
    Field f;
    uint64_t v = 0;
    while (fs.next(f, e)) {
        if (f.number == 2) {
            if (!expect_wire(f, kFixed64, m, e)) return false;
            std::memcpy(&x.error_std_dev, &f.value, 8);
        } else if (f.number == 1 || f.number == 3 || f.number == 4) {
            if (!scalar(f, m, v, e)) return false;
            v = (uint32_t)v;
            if (f.number == 1) x.p.lattice_dimension = (int64_t)v;
            else if (f.number == 3) x.p.plaintext_modulus_bits = (int32_t)std::min<uint64_t>(v, 1u << 30);
            else x.p.ciphertext_modulus_bits = (int32_t)std::min<uint64_t>(v, 1u << 30);
        }
    }
    return e.code == HECUDA_OK;
}

// SimplePIRParameters.native() (PirConversion.swift:416-460): errorStdDev must be one of ErrorStdDev's (3.2, 6.4) and
// the seed 32 bytes; the library's own parameter checks are the caller's (hecuda_simple_pir_params)
inline bool walk_params(const unsigned char *b, long long begin, long long end, Params &x, Error &e) {
    const char *m = "SimplePIRParameters";
    Fields fs{b, begin, end, m};
    Field f;
    bool seen_enc = false;
    uint64_t v = 0;
    x = Params{};
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!first_time(seen_enc, f, m, e)) return false;
            if (!walk_encryption_params(b, f.begin, f.end, x, e)) return false;
        } else if (f.number == 2) {
            if (!expect_wire(f, kLen, m, e)) return false;
            x.seed_begin = f.begin, x.seed_end = f.end;
        } else if (f.number >= 3 && f.number <= 6) {
            if (!scalar(f, m, v, e)) return false;
            const int64_t u = (int64_t)(uint32_t)v;
            if (f.number == 3) x.p.entry_size = u;
            else if (f.number == 4) x.p.entries_per_column = u;
            else if (f.number == 5) x.p.chunks_per_entry = u;
            else x.p.database_columns = u;
        }
    }
    if (e.code != HECUDA_OK) return false;
    if (x.error_std_dev != 3.2 && x.error_std_dev != 6.4)
        return e.invalid("invalidEncryptionParameters: Unsupported errorStdDev=" + std::to_string(x.error_std_dev) +
                         ", must be one of [3.2, 6.4]");
    if (x.seed_end - x.seed_begin != 32)
        return e.invalid("SimplePIRParameters: a_seed of " + std::to_string(x.seed_end - x.seed_begin) + " bytes, expected 32");
    x.p.error_std_dev = x.error_std_dev;
    x.p.word_bits = x.p.ciphertext_modulus_bits <= 32 ? 32 : 64;  // SimplePIRProcessDatabase/main.swift:369-371
    return true;
}

// SimplePIRConfig [0, size): counts in `shape`; with fill, every entry, chunk, parameter set and identifier range
struct Config {
    uint64_t chunk_size = 0;
    std::vector<uint64_t> original_index, size, chunk_count;  // per entry
    std::vector<std::pair<uint32_t, uint32_t>> chunks;         // (shard_index, index), entry-major
    std::vector<Params> params;
    std::vector<std::pair<long long, long long>> hint_ids;
    long long entry_count = 0, chunk_total = 0;
};

inline bool walk_entry(const unsigned char *b, long long begin, long long end, bool fill, Config &c, Error &e) {
    const char *m = "DatabaseMapping.Entry";
    Fields fs{b, begin, end, m};
    Field f;
    uint64_t index = 0, size = 0, chunks = 0, v = 0;
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!scalar(f, m, index, e)) return false;
        } else if (f.number == 2) {
            if (!scalar(f, m, size, e)) return false;
            size = (uint32_t)size;
        } else if (f.number == 3) {
            if (!expect_wire(f, kLen, m, e)) return false;
            uint32_t loc[2] = {0, 0};
            Fields lf{b, f.begin, f.end, "DatabaseMapping.ChunkLocation"};
            Field g;
            while (lf.next(g, e)) {
                if (g.number != 1 && g.number != 2) continue;
                if (!scalar(g, "DatabaseMapping.ChunkLocation", v, e)) return false;
                loc[g.number - 1] = (uint32_t)v;
            }
            if (e.code != HECUDA_OK) return false;
            ++chunks;
            if (fill) c.chunks.emplace_back(loc[0], loc[1]);
        }
    }
    if (e.code != HECUDA_OK) return false;
    ++c.entry_count;
    c.chunk_total += (long long)chunks;
    if (fill) c.original_index.push_back(index), c.size.push_back(size), c.chunk_count.push_back(chunks);
    return true;
}

inline bool walk_config(const unsigned char *b, long long size, bool fill, Config &c, Error &e) {
    const char *m = "SimplePIRConfig";
    c = Config{};
    Fields fs{b, 0, size, m};
    Field f;
    bool seen_map = false;
    while (fs.next(f, e)) {
        if (f.number == 1) {
            if (!first_time(seen_map, f, m, e)) return false;
            Fields mf{b, f.begin, f.end, "DatabaseMapping"};
            Field g;
            while (mf.next(g, e)) {
                if (g.number == 1) {
                    if (!expect_wire(g, kLen, "DatabaseMapping", e)) return false;
                    if (!walk_entry(b, g.begin, g.end, fill, c, e)) return false;
                } else if (g.number == 2) {
                    if (!scalar(g, "DatabaseMapping", c.chunk_size, e)) return false;
                    c.chunk_size = (uint32_t)c.chunk_size;
                }
            }
            if (e.code != HECUDA_OK) return false;
        } else if (f.number == 2) {
            if (!expect_wire(f, kLen, m, e)) return false;
            Params p;
            if (!walk_params(b, f.begin, f.end, p, e)) {
                e.what = "params " + std::to_string(c.params.size()) + ": " + e.what;
                return false;
            }
            c.params.push_back(p);
        } else if (f.number == 3) {
            if (!expect_wire(f, kLen, m, e)) return false;
            c.hint_ids.emplace_back(f.begin, f.end);
        }
    }
    return e.code == HECUDA_OK;
}

// SimplePIRParameters.proto() (PirConversion.swift:403-446)
inline Bytes encode_params(const hecuda_simple_pir_params &p, const unsigned char *seed) {
    Bytes enc, out;
    put_scalar(enc, 1, (uint32_t)p.lattice_dimension);
    if (p.error_std_dev != 0) {
        uint64_t bits = 0;
        std::memcpy(&bits, &p.error_std_dev, 8);
        put_key(enc, 2, kFixed64);
        for (int k = 0; k < 8; ++k) enc.push_back((unsigned char)(bits >> (8 * k)));
    }
    put_scalar(enc, 3, (uint32_t)p.plaintext_modulus_bits);
    put_scalar(enc, 4, (uint32_t)p.ciphertext_modulus_bits);
    put_message(out, 1, enc);
    put_message(out, 2, Bytes(seed, seed + 32));
    put_scalar(out, 3, (uint32_t)p.entry_size);
    put_scalar(out, 4, (uint32_t)p.entries_per_column);
    put_scalar(out, 5, (uint32_t)p.chunks_per_entry);
    put_scalar(out, 6, (uint32_t)p.database_columns);
    return out;
}

// SimplePIRConfig as the tool writes it (main.swift:231-240): the DatabaseMapping (DatabaseMap.proto(), :462-510),
// every shard's parameters, every hint identifier
inline Bytes encode_config(const uint64_t *original_index, const uint64_t *size, const uint64_t *chunk_count,
                           long long entry_count, const int64_t *chunks, uint64_t chunk_size,
                           const hecuda_simple_pir_params *params, const unsigned char *seeds, int shard_count,
                           const unsigned char *const *hint_ids, const uint64_t *hint_id_bytes, int hint_count) {
    Bytes mapping, out;
    long long at = 0;
    for (long long i = 0; i < entry_count; ++i) {
        Bytes entry;
        put_scalar(entry, 1, original_index[i]);
        put_scalar(entry, 2, (uint32_t)size[i]);
        for (uint64_t c = 0; c < chunk_count[i]; ++c, ++at) {
            Bytes loc;
            put_scalar(loc, 1, (uint32_t)chunks[2 * at]);
            put_scalar(loc, 2, (uint32_t)chunks[2 * at + 1]);
            put_message(entry, 3, loc);
        }
        put_message(mapping, 1, entry);
    }
    put_scalar(mapping, 2, (uint32_t)chunk_size);
    put_message(out, 1, mapping);
    for (int s = 0; s < shard_count; ++s) put_message(out, 2, encode_params(params[s], seeds + 32 * s));
    for (int h = 0; h < hint_count; ++h) put_message(out, 3, Bytes(hint_ids[h], hint_ids[h] + hint_id_bytes[h]));
    return out;
}

}  // namespace spirproto
}  // namespace hecuda
