// simple_pir_proto.cu -- the host-only C ABI of SimplePIR in the reference's protobuf messages (simple_pir_proto.hpp):
// the walk of a SimplePIRRequest, the client's framing of its request and reading of its response, and the
// SimplePIRConfig the SimplePIRProcessDatabase tool writes.  The device call that answers requests, and the size of its
// responses, are in simple_pir.cu (hecuda_simple_pir_compute_response_proto).
#include <algorithm>
#include <string>
#include <vector>

#include "capi_internal.hpp"
#include "simple_pir_proto.hpp"

using namespace hecuda;
using namespace hecuda::api;

namespace {

int32_t copy_out(const proto::Bytes &msg, uint8_t *out, uint64_t capacity, uint64_t *written) {
    *written = msg.size();
    if (!out) return HECUDA_OK;
    if (capacity < msg.size())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below " + std::to_string(msg.size()));
    std::copy(msg.begin(), msg.end(), out);
    return HECUDA_OK;
}

// the config's walk and every refusal of SimplePIRParameters.native() and of the library's parameters
int32_t walk_config(const uint8_t *bytes, uint64_t byte_count, bool fill, spirproto::Config &c) {
    if (!bytes && byte_count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Error e;
    if (!spirproto::walk_config(bytes, (long long)byte_count, fill, c, e)) return fail(e.code, e.what);
    for (size_t s = 0; s < c.params.size(); ++s) {
        int64_t m, k, scalars;
        u64 p;
        const int32_t rc = simple_pir_derive(&c.params[s].p, m, k, scalars, p);
        if (rc) return fail(rc, "params " + std::to_string(s) + ": " + std::string(last_error_cstr()));
    }
    return HECUDA_OK;
}

int32_t config_bytes(const uint64_t *original_indices, const uint64_t *sizes, const uint64_t *chunk_counts, int64_t entry_count,
                     const int64_t *chunk_locations, uint64_t chunk_size, const hecuda_simple_pir_params *params,
                     const uint8_t *seeds, int32_t shard_count, const uint8_t *const *hint_ids, const uint64_t *hint_id_bytes,
                     int32_t hint_count, proto::Bytes &out) {
    if (entry_count < 0 || shard_count < 0 || hint_count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative count");
    if ((entry_count && (!original_indices || !sizes || !chunk_counts)) || (shard_count && (!params || !seeds)) ||
        (hint_count && (!hint_ids || !hint_id_bytes)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    uint64_t chunks = 0;
    for (int64_t i = 0; i < entry_count; ++i) chunks += chunk_counts[i];
    if (chunks && !chunk_locations) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    for (int32_t h = 0; h < hint_count; ++h)
        if (hint_id_bytes[h] && !hint_ids[h]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    out = spirproto::encode_config(original_indices, sizes, chunk_counts, entry_count, chunk_locations, chunk_size, params,
                                   seeds, shard_count, hint_ids, hint_id_bytes, hint_count);
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_simple_pir_request_fields_read(const uint8_t *bytes, uint64_t byte_count,
                                              hecuda_simple_pir_request_fields *fields) {
    if (!fields || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Error e;
    spirproto::Request r;
    if (!spirproto::walk_request(bytes, (long long)byte_count, r, e)) return fail(e.code, e.what);
    *fields = hecuda_simple_pir_request_fields{};
    fields->has_request = r.has_request;
    fields->row_count = r.matrix.rows;
    fields->col_count = r.matrix.columns;
    fields->shard_index = r.shard_index;
    fields->data_run_count = (int64_t)r.matrix.runs.size();
    for (const auto &run : r.matrix.runs) fields->data_bytes += (uint64_t)(run.second - run.first);
    fields->configuration_hash_offset = (uint64_t)r.hash_begin;
    fields->configuration_hash_bytes = (uint64_t)(r.hash_end - r.hash_begin);
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_request_write(uint32_t row_count, uint32_t col_count, const uint64_t *data, uint32_t shard_index,
                                        const uint8_t *configuration_hash, uint64_t hash_bytes, uint8_t *out,
                                        uint64_t capacity, uint64_t *written) {
    const long long values = (long long)row_count * col_count;
    if (!written || (values && !data) || (hash_bytes && !configuration_hash))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Bytes msg;
    proto::put_message(msg, 1, spirproto::encode_matrix(row_count, col_count, data, values));
    proto::put_scalar(msg, 2, shard_index);
    if (hash_bytes) proto::put_message(msg, 3, proto::Bytes(configuration_hash, configuration_hash + hash_bytes));
    return copy_out(msg, out, capacity, written);
}

int32_t hecuda_simple_pir_response_read(const uint8_t *bytes, uint64_t byte_count, uint32_t *row_count, uint32_t *col_count,
                                        uint64_t *data, int64_t capacity) {
    if (!row_count || !col_count || (!bytes && byte_count) || capacity < 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Error e;
    spirproto::Response r;
    if (!spirproto::walk_response(bytes, (long long)byte_count, (size_t)capacity, r, e)) return fail(e.code, e.what);
    if (!r.has_response) return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePIRResponse.response is not set");
    *row_count = r.rows, *col_count = r.columns;
    if (!r.data.empty() && !data) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    std::copy(r.data.begin(), r.data.end(), data);
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_config_describe(const uint8_t *bytes, uint64_t byte_count, hecuda_simple_pir_config_shape *shape) {
    if (!shape) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    spirproto::Config c;
    const int32_t rc = walk_config(bytes, byte_count, false, c);
    if (rc) return rc;
    shape->entry_count = c.entry_count;
    shape->chunk_count = c.chunk_total;
    shape->chunk_size = c.chunk_size;
    shape->shard_count = (int32_t)c.params.size();
    shape->hint_identifier_count = (int32_t)c.hint_ids.size();
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_config_read(const uint8_t *bytes, uint64_t byte_count, uint64_t *original_indices, uint64_t *sizes,
                                      uint64_t *chunk_counts, int64_t *chunk_locations, hecuda_simple_pir_params *params,
                                      uint8_t *seeds, uint64_t *hint_identifier_ranges) {
    spirproto::Config c;
    const int32_t rc = walk_config(bytes, byte_count, true, c);
    if (rc) return rc;
    if ((c.entry_count && (!original_indices || !sizes || !chunk_counts)) || (c.chunk_total && !chunk_locations) ||
        (!c.params.empty() && (!params || !seeds)) || (!c.hint_ids.empty() && !hint_identifier_ranges))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    std::copy(c.original_index.begin(), c.original_index.end(), original_indices);
    std::copy(c.size.begin(), c.size.end(), sizes);
    std::copy(c.chunk_count.begin(), c.chunk_count.end(), chunk_counts);
    for (size_t i = 0; i < c.chunks.size(); ++i) {
        chunk_locations[2 * i] = c.chunks[i].first;
        chunk_locations[2 * i + 1] = c.chunks[i].second;
    }
    for (size_t s = 0; s < c.params.size(); ++s) {
        params[s] = c.params[s].p;
        std::copy(bytes + c.params[s].seed_begin, bytes + c.params[s].seed_end, seeds + 32 * s);
    }
    for (size_t h = 0; h < c.hint_ids.size(); ++h) {
        hint_identifier_ranges[2 * h] = (uint64_t)c.hint_ids[h].first;
        hint_identifier_ranges[2 * h + 1] = (uint64_t)(c.hint_ids[h].second - c.hint_ids[h].first);
    }
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_config_serialized_byte_count(const uint64_t *original_indices, const uint64_t *sizes,
                                                       const uint64_t *chunk_counts, int64_t entry_count,
                                                       const int64_t *chunk_locations, uint64_t chunk_size,
                                                       const hecuda_simple_pir_params *params, const uint8_t *seeds,
                                                       int32_t shard_count, const uint8_t *const *hint_identifiers,
                                                       const uint64_t *hint_identifier_bytes, int32_t hint_count,
                                                       uint64_t *bytes) {
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Bytes msg;
    const int32_t rc = config_bytes(original_indices, sizes, chunk_counts, entry_count, chunk_locations, chunk_size, params,
                                    seeds, shard_count, hint_identifiers, hint_identifier_bytes, hint_count, msg);
    if (rc) return rc;
    *bytes = msg.size();
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_config_serialize(const uint64_t *original_indices, const uint64_t *sizes,
                                           const uint64_t *chunk_counts, int64_t entry_count, const int64_t *chunk_locations,
                                           uint64_t chunk_size, const hecuda_simple_pir_params *params, const uint8_t *seeds,
                                           int32_t shard_count, const uint8_t *const *hint_identifiers,
                                           const uint64_t *hint_identifier_bytes, int32_t hint_count, uint8_t *out,
                                           uint64_t capacity) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    proto::Bytes msg;
    const int32_t rc = config_bytes(original_indices, sizes, chunk_counts, entry_count, chunk_locations, chunk_size, params,
                                    seeds, shard_count, hint_identifiers, hint_identifier_bytes, hint_count, msg);
    if (rc) return rc;
    uint64_t written = 0;
    return copy_out(msg, out, capacity, &written);
}

}  // extern "C"
