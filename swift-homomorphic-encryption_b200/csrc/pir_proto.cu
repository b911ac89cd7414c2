// pir_proto.cu -- the host-only C ABI of PIR in the reference's protobuf messages (pir_proto.hpp): the walk of a
// PIRRequest, the size of a PIRResponse, and the client's framing of its query and key and reading of its reply.  The
// device calls that answer the messages are in pir.cu (hecuda_mulpir_compute_response_clients_proto) and capi.cu
// (hecuda_evk_create_proto_many).
#include <algorithm>
#include <string>
#include <vector>

#include "capi_internal.hpp"
#include "pir_proto.hpp"

using namespace hecuda;
using namespace hecuda::api;

namespace {

// the sizes of polynomials over `rows` rows from `base` (the query's L rows, a key's L + 1, a reply's one)
int32_t sizes(const hecuda_context *h, int32_t base, int32_t rows, pirproto::PolySizes &sz) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    NttRowMap map;
    CodecConsts cc;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err) || !codec_consts(*h->ctx, map, 0, cc, err))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    sz = pirproto::poly_sizes(cc, h->ctx->n);
    return HECUDA_OK;
}

int32_t emit(const pirproto::Bytes &bytes, uint8_t *out, uint64_t capacity, uint64_t *written) {
    if (!written) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *written = bytes.size();
    if (!out) return HECUDA_OK;
    if (capacity < bytes.size())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below " + std::to_string(bytes.size()));
    std::copy(bytes.begin(), bytes.end(), out);
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_pir_request_fields_read(const uint8_t *bytes, uint64_t byte_count, hecuda_pir_request_fields *out) {
    if (!out || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pirproto::Error e;
    hecuda_pir_request_fields r;
    if (!pirproto::walk_pir_request(bytes, (long long)byte_count, r, e)) return fail(e.code, e.what);
    *out = r;
    return HECUDA_OK;
}

int32_t hecuda_mulpir_response_proto_byte_count(const hecuda_context *h, int32_t chunk_count, int32_t indices_count,
                                                int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint64_t *bytes) {
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (chunk_count < 1 || indices_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid PIR parameter");
    pirproto::PolySizes sz;
    int32_t rc = sizes(h, HECUDA_BASE_Q, 1, sz);
    if (rc) return rc;
    const long long b0 = sz.bytes(skip_lsbs_poly0), b1 = sz.bytes(skip_lsbs_poly1);
    if (b0 < 0 || b1 < 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCoefficientPacking(skipLSBs: " +
                                                     std::to_string(b0 < 0 ? skip_lsbs_poly0 : skip_lsbs_poly1) + ")");
    *bytes = (uint64_t)pirproto::place_response(indices_count, chunk_count, b0, b1, skip_lsbs_poly0, skip_lsbs_poly1).size;
    return HECUDA_OK;
}

int32_t hecuda_pir_encrypted_indices_write(const hecuda_context *h, const uint8_t *poly0, const uint8_t *seeds,
                                           int32_t ciphertext_count, int32_t indices_count, uint8_t *out, uint64_t capacity,
                                           uint64_t *written) {
    pirproto::PolySizes sz;
    int32_t rc = sizes(h, HECUDA_BASE_Q, h ? h->ctx->L : 0, sz);
    if (rc) return rc;
    if (ciphertext_count < 0 || indices_count < 0 || (ciphertext_count && (!poly0 || !seeds)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    return emit(pirproto::encode_encrypted_indices(poly0, seeds, ciphertext_count, sz.bytes(0), (uint64_t)indices_count), out,
                capacity, written);
}

int32_t hecuda_pir_evaluation_key_write(const hecuda_context *h, const uint8_t *relin_poly0, const uint8_t *relin_seeds,
                                        const uint32_t *elements, int32_t element_count, const uint8_t *galois_poly0,
                                        const uint8_t *galois_seeds, uint8_t *out, uint64_t capacity, uint64_t *written) {
    pirproto::PolySizes sz;
    int32_t rc = sizes(h, HECUDA_BASE_KEYSWITCH, h ? h->ctx->L + 1 : 0, sz);
    if (rc) return rc;
    if ((relin_poly0 == nullptr) != (relin_seeds == nullptr) || element_count < 0 ||
        (element_count && (!elements || !galois_poly0 || !galois_seeds)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const long long L = h->ctx->L, bytes = sz.bytes(0);
    pirproto::Bytes map, key;
    for (int32_t g = 0; g < element_count; ++g) {  // map entry { 1 key, 2 value }
        pirproto::Bytes entry;
        pirproto::put_scalar(entry, 1, elements[g]);
        pirproto::put_message(entry, 2, pirproto::encode_key_switch_key(galois_poly0 + g * L * bytes, galois_seeds + g * L * 32,
                                                                        L, bytes));
        pirproto::put_message(map, 1, entry);
    }
    if (element_count) pirproto::put_message(key, 1, map);
    if (relin_poly0) {
        pirproto::Bytes relin;
        pirproto::put_message(relin, 1, pirproto::encode_key_switch_key(relin_poly0, relin_seeds, L, bytes));
        pirproto::put_message(key, 2, relin);
    }
    return emit(key, out, capacity, written);
}

int32_t hecuda_pir_response_read(const hecuda_context *h, const uint8_t *bytes, uint64_t byte_count, int32_t chunk_count,
                                 int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                 uint64_t *poly_offsets) {
    pirproto::PolySizes sz;
    int32_t rc = sizes(h, HECUDA_BASE_Q, 1, sz);
    if (rc) return rc;
    if ((!bytes && byte_count) || !poly_offsets) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pirproto::Error e;
    std::vector<long long> at;
    if (!pirproto::walk_pir_response(bytes, (long long)byte_count, sz, indices_count, chunk_count, skip_lsbs_poly0,
                                     skip_lsbs_poly1, at, e))
        return fail(e.code, e.what);
    std::copy(at.begin(), at.end(), poly_offsets);
    return HECUDA_OK;
}

}  // extern "C"
