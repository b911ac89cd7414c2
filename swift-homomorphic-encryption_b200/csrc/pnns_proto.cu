// pnns_proto.cu -- the host-only C ABI of PNNS in the reference's protobuf messages (pnns_proto.hpp): the walk of a
// PNNSRequest, and the client's framing of its request and reading of its shard response.  The device call that
// answers the messages, and the response size, are in pnns.cu (hecuda_pnns_compute_response_clients_proto).
#include <algorithm>
#include <string>
#include <vector>

#include "capi_internal.hpp"
#include "pnns_proto.hpp"

using namespace hecuda;
using namespace hecuda::api;

namespace {

// the sizes of polynomials over the first `rows` q rows of every context (the query's L, a reply's one)
int32_t context_sizes(const hecuda_context *const *ctxs, int32_t count, bool reply, std::vector<pnnsproto::PolySizes> &out) {
    if (!ctxs || count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    out.assign((size_t)count, pnnsproto::PolySizes{});
    for (int32_t k = 0; k < count; ++k) {
        int32_t rc = check_ctx(ctxs[k]);
        if (rc) return rc;
        const Context &c = *ctxs[k]->ctx;
        NttRowMap map;
        CodecConsts cc;
        std::string err;
        if (!make_map(c, HECUDA_BASE_Q, reply ? 1 : c.L, map, err) || !codec_consts(c, map, 0, cc, err))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
        out[(size_t)k] = pnnsproto::poly_sizes(cc, c.n);
    }
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_pnns_request_fields_read(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_request_fields *fields,
                                        uint32_t *shard_indices, int64_t index_capacity, uint64_t *shard_id_ranges,
                                        int64_t id_capacity) {
    if (!fields || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsproto::Error e;
    pnnsproto::Request r;
    if (!pnnsproto::walk_pnns_request(bytes, (long long)byte_count, r, e)) return fail(e.code, e.what);
    if ((shard_indices && index_capacity < (int64_t)r.shard_indices.size()) ||
        (shard_id_ranges && id_capacity < (int64_t)r.shard_ids.size()))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity below the request's " + std::to_string(r.shard_indices.size()) +
                                                     " shard indices and " + std::to_string(r.shard_ids.size()) + " shard ids");
    for (size_t i = 0; shard_indices && i < r.shard_indices.size(); ++i) shard_indices[i] = (uint32_t)r.shard_indices[i];
    for (size_t i = 0; shard_id_ranges && i < r.shard_ids.size(); ++i) {
        shard_id_ranges[2 * i] = (uint64_t)r.shard_ids[i].first;
        shard_id_ranges[2 * i + 1] = (uint64_t)(r.shard_ids[i].second - r.shard_ids[i].first);
    }
    *fields = r.fields;
    return HECUDA_OK;
}

int32_t hecuda_pnns_request_write(const hecuda_context *const *ctxs, int32_t count, uint32_t row_count, uint32_t column_count,
                                  const uint8_t *const *poly0, const uint8_t *const *seeds, int32_t ciphertext_count,
                                  const uint8_t *config_id, uint64_t config_id_bytes, const uint8_t *evaluation_key,
                                  uint64_t evaluation_key_bytes, uint64_t key_timestamp, const uint8_t *key_identifier,
                                  uint64_t key_identifier_bytes, uint8_t *out, uint64_t capacity, uint64_t *written) {
    std::vector<pnnsproto::PolySizes> sizes;
    int32_t rc = context_sizes(ctxs, count, false, sizes);
    if (rc) return rc;
    if (!written || ciphertext_count < 0 || (ciphertext_count && (!poly0 || !seeds)) || (config_id_bytes && !config_id) ||
        (evaluation_key_bytes && !evaluation_key) || (key_identifier_bytes && !key_identifier))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsproto::Bytes msg;
    for (int32_t k = 0; k < count; ++k) {  // Query.proto(): one SerializedCiphertextMatrix per plaintext modulus
        if (ciphertext_count && (!poly0[k] || !seeds[k])) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
        pnnsproto::put_message(msg, 2, pnnsproto::encode_query_matrix(row_count, column_count, poly0[k], seeds[k],
                                                                      ciphertext_count, sizes[(size_t)k].bytes(0)));
    }
    if (config_id_bytes) {
        pnnsproto::put_key(msg, 4, pnnsproto::kLen);
        pnnsproto::put_varint(msg, config_id_bytes);
        msg.insert(msg.end(), config_id, config_id + config_id_bytes);
    }
    if (evaluation_key) {  // api.shared.v1.EvaluationKey { 1 metadata { 1 timestamp  2 identifier }  2 evaluation_key }
        pnnsproto::Bytes metadata, key, inner(evaluation_key, evaluation_key + evaluation_key_bytes);
        pnnsproto::put_scalar(metadata, 1, key_timestamp);
        if (key_identifier_bytes) {
            pnnsproto::put_key(metadata, 2, pnnsproto::kLen);
            pnnsproto::put_varint(metadata, key_identifier_bytes);
            metadata.insert(metadata.end(), key_identifier, key_identifier + key_identifier_bytes);
        }
        pnnsproto::put_message(key, 1, metadata);
        pnnsproto::put_message(key, 2, inner);
        pnnsproto::put_message(msg, 5, key);
    }
    *written = msg.size();
    if (!out) return HECUDA_OK;
    if (capacity < msg.size())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below " + std::to_string(msg.size()));
    std::copy(msg.begin(), msg.end(), out);
    return HECUDA_OK;
}

int32_t hecuda_pnns_shard_response_read(const hecuda_context *const *ctxs, int32_t count, const uint8_t *bytes,
                                        uint64_t byte_count, hecuda_pnns_shard_response_shape *shape, uint64_t *poly_offsets,
                                        int32_t *skip_lsbs, uint64_t *entry_ids, uint64_t *metadata_ranges) {
    std::vector<pnnsproto::PolySizes> sizes;
    int32_t rc = context_sizes(ctxs, count, true, sizes);
    if (rc) return rc;
    if (!shape || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsproto::Error e;
    pnnsproto::ShardResponse r;
    if (!pnnsproto::walk_shard_response(bytes, (long long)byte_count, sizes, r, e)) return fail(e.code, e.what);
    // the reply count of a .denseColumn result of database rows x query rows (PlaintextMatrix.mulTranspose(matrix:))
    const long long n = sizes[0].n, half = n / 2;
    if (r.rows == 0 || r.columns == 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions(rowCount: " + std::to_string(r.rows) +
                                                     ", columnCount: " + std::to_string(r.columns) + ")");
    const long long S = half / (long long)r.rows, G = S > 0 ? ((long long)r.columns + S - 1) / S : 0;
    const long long expected = S > 0 ? (G + 1) / 2 : (long long)r.columns * (((long long)r.rows + n - 1) / n);
    if (r.replies != expected)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongCiphertextCount(got: " + std::to_string(r.replies) + ", expected: " +
                                                     std::to_string(expected) + ")");
    shape->matrix_count = count;
    shape->reply_count = (int32_t)r.replies;
    shape->row_count = (uint32_t)r.rows, shape->column_count = (uint32_t)r.columns;
    shape->id_count = (int64_t)r.ids.size(), shape->metadata_count = (int64_t)r.metadata.size();
    for (int32_t k = 0; k < count; ++k) {
        for (long long i = 0; poly_offsets && i < r.replies; ++i)
            poly_offsets[(size_t)k * r.replies + i] = (uint64_t)r.poly_at[(size_t)k][(size_t)i];
        if (skip_lsbs) skip_lsbs[2 * k] = r.skip[(size_t)k][0], skip_lsbs[2 * k + 1] = r.skip[(size_t)k][1];
    }
    if (entry_ids) std::copy(r.ids.begin(), r.ids.end(), entry_ids);
    for (size_t i = 0; metadata_ranges && i < r.metadata.size(); ++i) {
        metadata_ranges[2 * i] = (uint64_t)r.metadata[i].first;
        metadata_ranges[2 * i + 1] = (uint64_t)(r.metadata[i].second - r.metadata[i].first);
    }
    return HECUDA_OK;
}

}  // extern "C"
