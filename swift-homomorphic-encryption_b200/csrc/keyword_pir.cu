// keyword_pir.cu -- keyword PIR's data-parallel half on the device (KeywordPir/HashBucket.swift, CuckooTable.swift,
// KeywordPirProtocol.swift:191-247):
//
//   keyword_hash_kernel       HashKeyword.hash of every keyword, one thread each
//   hash_indices_kernel       HashKeyword.hashIndices of every row for one bucketsPerTable, one thread each; launched
//                             once per bucket count the placement (cuckoo.hpp, on the host) reaches
//   bucket_serialize_kernel   HashBucket.serialize of every bucket from the placement's CSR, one warp each
//
// The index arithmetic is in keyword_pir.cuh.  Each table's slice of the serialized buckets goes straight into the
// MulPir packing and Eval conversion (pir.cu, process_db.cu): bucket bytes never cross PCIe.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "capi_internal.hpp"
#include "cuckoo.hpp"
#include "keyword_pir.cuh"

using namespace hecuda;
using namespace hecuda::api;

struct hecuda_cuckoo_table {
    const hecuda_context *owner = nullptr;
    cuckoo::Config config{};
    int64_t count = 0;                     // rows given
    int64_t bucket_count = 0, buckets_per_table = 0;
    std::vector<uint64_t> offsets;         // bucket_count + 1 serialized-byte offsets
    hecuda_cuckoo_summary summary{};
    unsigned char *d_values = nullptr;     // the rows' values, uploaded once
    uint64_t *d_value_offsets = nullptr;   // count + 1
    uint64_t *d_hashes = nullptr;          // count keyword hashes
    int64_t *d_row_ptr = nullptr;          // bucket_count + 1: bucket b's entries are d_ids[d_row_ptr[b] .. d_row_ptr[b+1])
    int64_t *d_ids = nullptr;              // entry ids in slot order
    uint64_t *d_offsets = nullptr;         // `offsets` on the device
};

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) keyword_hash_kernel(const unsigned char *__restrict__ keywords,
                                                               const uint64_t *__restrict__ offsets, long long count,
                                                               uint64_t *__restrict__ hashes) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= count) return;
    hashes[i] = kwpir::keyword_hash(keywords + offsets[i], (long long)(offsets[i + 1] - offsets[i]));
}

__global__ void __launch_bounds__(kThreads) hash_indices_kernel(const uint64_t *__restrict__ hashes, long long count,
                                                               long long bucket_count, int h, int64_t *__restrict__ out) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= count) return;
    kwpir::hash_indices(hashes[i], bucket_count, h, out + i * h);
}

// One warp per bucket: lane 0 writes the slot count, then the warp writes each slot's bytes in turn.
__global__ void __launch_bounds__(kThreads) bucket_serialize_kernel(long long buckets, const int64_t *__restrict__ row_ptr,
                                                                   const int64_t *__restrict__ ids,
                                                                   const uint64_t *__restrict__ hashes,
                                                                   const unsigned char *__restrict__ values,
                                                                   const uint64_t *__restrict__ value_offsets,
                                                                   const uint64_t *__restrict__ out_offsets,
                                                                   unsigned char *__restrict__ out) {
    const long long b = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= buckets) return;
    unsigned char *dst = out + out_offsets[b];
    const long long first = row_ptr[b], last = row_ptr[b + 1];
    if (lane == 0) dst[0] = (unsigned char)(last - first);
    long long at = 1;
    for (long long k = first; k < last; ++k) {
        const long long e = ids[k];
        const uint64_t hash = hashes[e];
        const unsigned char *value = values + value_offsets[e];
        const long long length = (long long)(value_offsets[e + 1] - value_offsets[e]);
        const long long size = kwpir::slot_size(length);
        for (long long j = lane; j < size; j += 32) dst[at + j] = (unsigned char)kwpir::slot_byte(hash, value, length, j);
        at += size;
    }
}

unsigned grid_for(long long items, long long per_block) { return (unsigned)((items + per_block - 1) / per_block); }

cudaError_t launch_keyword_hash(const unsigned char *d_keywords, const uint64_t *d_offsets, int64_t count, uint64_t *d_hashes) {
    if (count == 0) return cudaSuccess;
    return launch(keyword_hash_kernel, grid_for(count, kThreads), kThreads, 0, 0, d_keywords, d_offsets, count, d_hashes);
}

cudaError_t launch_hash_indices(const uint64_t *d_hashes, int64_t count, int64_t bucket_count, int h, int64_t *d_out) {
    if (count == 0) return cudaSuccess;
    return launch(hash_indices_kernel, grid_for(count, kThreads), kThreads, 0, 0, d_hashes, count, bucket_count, h, d_out);
}

// Bucket bytes into d_out (table->offsets.back() bytes) on the default stream
cudaError_t launch_bucket_serialize(const hecuda_cuckoo_table *t, unsigned char *d_out) {
    if (t->bucket_count == 0) return cudaSuccess;
    return launch(bucket_serialize_kernel, grid_for(t->bucket_count * 32, kThreads), kThreads, 0, 0, t->bucket_count, t->d_row_ptr,
                  t->d_ids, t->d_hashes, t->d_values, t->d_value_offsets, t->d_offsets, d_out);
}

int32_t have_device() {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    return HECUDA_OK;
}

// offsets[0..count] must not decrease; `longest` gets the longest row
int32_t check_offsets(const uint64_t *offsets, int64_t count, uint64_t &longest, const char *what) {
    longest = 0;
    for (int64_t i = 0; i < count; ++i) {
        if (offsets[i + 1] < offsets[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, std::string(what) + " offsets must not decrease");
        longest = std::max<uint64_t>(longest, offsets[i + 1] - offsets[i]);
    }
    return HECUDA_OK;
}

template <class T>
cudaError_t upload_new(T **dst, const void *src, size_t bytes) {
    cudaError_t e = cudaMalloc(dst, std::max<size_t>(bytes, 1));
    if (e == cudaSuccess && bytes) e = upload(*dst, src, bytes);
    return e;
}

// Uploads the keywords, hashes them on the device, and leaves the hashes in *d_hashes (device) and `hashes` (host).
cudaError_t hash_keywords(const uint8_t *keywords, const uint64_t *offsets, int64_t count, uint64_t **d_hashes,
                          uint64_t *hashes) {
    unsigned char *d_keywords = nullptr;
    uint64_t *d_offsets = nullptr;
    cudaError_t e = upload_new(&d_keywords, keywords, (size_t)offsets[count]);
    if (e == cudaSuccess) e = upload_new(&d_offsets, offsets, (size_t)(count + 1) * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(d_hashes, (size_t)std::max<int64_t>(count, 1) * sizeof(uint64_t));
    if (e == cudaSuccess) e = launch_keyword_hash(d_keywords, d_offsets, count, *d_hashes);
    if (e == cudaSuccess && count) e = cudaMemcpy(hashes, *d_hashes, (size_t)count * sizeof(uint64_t), cudaMemcpyDeviceToHost);
    cudaFree(d_offsets);
    cudaFree(d_keywords);
    return e;
}

void free_table(hecuda_cuckoo_table *t) {
    if (!t) return;
    cudaFree(t->d_values);
    cudaFree(t->d_value_offsets);
    cudaFree(t->d_hashes);
    cudaFree(t->d_row_ptr);
    cudaFree(t->d_ids);
    cudaFree(t->d_offsets);
    delete t;
}

}  // namespace

extern "C" {

int32_t hecuda_keyword_hash(const uint8_t *keywords, const uint64_t *offsets, int64_t count, uint64_t *hashes) {
    if (!keywords || !offsets || !hashes || count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    uint64_t longest = 0;
    int32_t rc = check_offsets(offsets, count, longest, "keyword");
    if (!rc) rc = have_device();
    if (rc) return rc;
    uint64_t *d_hashes = nullptr;
    cudaError_t e = hash_keywords(keywords, offsets, count, &d_hashes, hashes);
    cudaFree(d_hashes);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "keyword hash");
}

int32_t hecuda_keyword_hash_indices(const uint64_t *hashes, int64_t count, int64_t bucket_count,
                                    int32_t hash_function_count, int64_t *out) {
    if (!hashes || !out || count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    if (bucket_count < 1 || hash_function_count < 1)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "bucket count and hash function count must be positive");
    int32_t rc = have_device();
    if (rc) return rc;
    const size_t words = (size_t)count * hash_function_count;
    uint64_t *d_hashes = nullptr;
    int64_t *d_out = nullptr;
    cudaError_t e = upload_new(&d_hashes, hashes, (size_t)count * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&d_out, std::max<size_t>(words, 1) * sizeof(int64_t));
    if (e == cudaSuccess) e = launch_hash_indices(d_hashes, count, bucket_count, hash_function_count, d_out);
    if (e == cudaSuccess && words) e = cudaMemcpy(out, d_out, words * sizeof(int64_t), cudaMemcpyDeviceToHost);
    cudaFree(d_out);
    cudaFree(d_hashes);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "keyword hash indices");
}

int32_t hecuda_cuckoo_table_create(const hecuda_context *h, const uint8_t *keywords, const uint64_t *keyword_offsets,
                                   const uint8_t *values, const uint64_t *value_offsets, int64_t count,
                                   const hecuda_cuckoo_config *config, int32_t rng, uint64_t seed,
                                   hecuda_cuckoo_table **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!keywords || !keyword_offsets || !values || !value_offsets || !config || count < 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    const cuckoo::Config c{config->hash_function_count, config->max_eviction_count, config->max_serialized_bucket_size,
                           config->slot_count,          config->multiple_tables != 0, config->fixed_bucket_count,
                           config->expansion_factor,    config->target_load_factor};
    if (config->fixed_bucket_count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCuckooConfig");
    const std::string invalid = cuckoo::validate(c);
    if (!invalid.empty()) return fail(HECUDA_ERR_INVALID_ARGUMENT, invalid);
    if (rng != HECUDA_CUCKOO_RNG_COUNTER && rng != HECUDA_CUCKOO_RNG_SPLITMIX64)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "unknown cuckoo rng " + std::to_string(rng));
    uint64_t longest_keyword = 0, longest_value = 0;
    rc = check_offsets(keyword_offsets, count, longest_keyword, "keyword");
    if (!rc) rc = check_offsets(value_offsets, count, longest_value, "value");
    if (rc) return rc;
    if (longest_value > (uint64_t)kwpir::kMaxValueSize)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidHashBucketEntryValueSize(maxSize: 65535)");

    hecuda_cuckoo_table *t = new (std::nothrow) hecuda_cuckoo_table();
    if (!t) return fail(HECUDA_ERR_CUDA, "out of host memory");
    t->owner = h;
    t->config = c;
    t->count = count;
    const int hf = c.hash_function_count;
    std::vector<uint64_t> hashes((size_t)count);
    std::vector<int64_t> candidates((size_t)count * hf);
    int64_t *d_candidates = nullptr;
    cudaError_t e = hash_keywords(keywords, keyword_offsets, count, &t->d_hashes, hashes.data());
    if (e == cudaSuccess) e = upload_new(&t->d_values, values, (size_t)value_offsets[count]);
    if (e == cudaSuccess) e = upload_new(&t->d_value_offsets, value_offsets, (size_t)(count + 1) * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&d_candidates, std::max<size_t>(candidates.size(), 1) * sizeof(int64_t));
    if (e != cudaSuccess) {
        cudaFree(d_candidates);
        free_table(t);
        return cuda_fail(e, "cuckoo table upload");
    }
    // HashKeyword.hashIndices of every row for one bucketsPerTable
    auto candidates_for = [&](int64_t per_table) -> const int64_t * {
        cudaError_t ce = launch_hash_indices(t->d_hashes, count, per_table, hf, d_candidates);
        if (ce == cudaSuccess && count)
            ce = cudaMemcpy(candidates.data(), d_candidates, candidates.size() * sizeof(int64_t), cudaMemcpyDeviceToHost);
        if (ce != cudaSuccess) throw ce;
        return candidates.data();
    };
    cuckoo::Table<decltype(candidates_for)> table(c, count, keywords, keyword_offsets, hashes.data(), value_offsets,
                                                  cuckoo::Generator{rng, seed}, candidates_for);
    std::string failure;
    try {
        table.build();
    } catch (const cuckoo::Failure &f) {
        failure = f.message;
    } catch (cudaError_t ce) {
        e = ce;
    }
    cudaFree(d_candidates);
    if (!failure.empty() || e != cudaSuccess) {
        free_table(t);
        return failure.empty() ? cuda_fail(e, "cuckoo table candidates") : fail(HECUDA_ERR_INVALID_ARGUMENT, failure);
    }

    // the placement as CSR, and every bucket's byte offset (the sizes were tracked during placement)
    const std::vector<cuckoo::Bucket> &buckets = table.buckets();
    t->bucket_count = (int64_t)buckets.size();
    t->buckets_per_table = table.buckets_per_table();
    std::vector<int64_t> row_ptr(buckets.size() + 1, 0), ids;
    t->offsets.assign(buckets.size() + 1, 0);
    hecuda_cuckoo_summary &s = t->summary;
    for (size_t b = 0; b < buckets.size(); ++b) {
        const cuckoo::Bucket &bucket = buckets[b];
        ids.insert(ids.end(), bucket.slots.begin(), bucket.slots.end());
        row_ptr[b + 1] = (int64_t)ids.size();
        t->offsets[b + 1] = t->offsets[b] + (uint64_t)bucket.size;
        s.empty_bucket_count += bucket.slots.empty() ? 1 : 0;
        s.max_serialized_bucket_size = std::max(s.max_serialized_bucket_size, bucket.size);
    }
    s.entry_count = (int64_t)ids.size();
    s.bucket_count = t->bucket_count;
    s.buckets_per_table = t->buckets_per_table;
    s.serialized_bytes = (int64_t)t->offsets.back();
    e = upload_new(&t->d_row_ptr, row_ptr.data(), row_ptr.size() * sizeof(int64_t));
    if (e == cudaSuccess) e = upload_new(&t->d_ids, ids.data(), ids.size() * sizeof(int64_t));
    if (e == cudaSuccess) e = upload_new(&t->d_offsets, t->offsets.data(), t->offsets.size() * sizeof(uint64_t));
    if (e != cudaSuccess) {
        free_table(t);
        return cuda_fail(e, "cuckoo table placement upload");
    }
    *out = t;
    return HECUDA_OK;
}

int32_t hecuda_cuckoo_table_summarize(const hecuda_cuckoo_table *t, hecuda_cuckoo_summary *out) {
    if (!t || !out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = t->summary;
    return HECUDA_OK;
}

int32_t hecuda_cuckoo_table_serialize_buckets(const hecuda_cuckoo_table *t, uint8_t *bytes, uint64_t capacity,
                                              uint64_t *offsets) {
    if (!t || !bytes || !offsets) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const uint64_t total = t->offsets.back();
    if (capacity < total) return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity below the serialized bucket bytes");
    int32_t rc = check_ctx(t->owner);
    if (rc) return rc;
    unsigned char *d_bytes = nullptr;
    cudaError_t e = cudaMalloc(&d_bytes, std::max<uint64_t>(total, 1));
    if (e == cudaSuccess) e = launch_bucket_serialize(t, d_bytes);
    if (e == cudaSuccess && total) e = cudaMemcpy(bytes, d_bytes, total, cudaMemcpyDeviceToHost);
    cudaFree(d_bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cuckoo table serialize");
    std::memcpy(offsets, t->offsets.data(), t->offsets.size() * sizeof(uint64_t));
    return HECUDA_OK;
}

int32_t hecuda_cuckoo_table_destroy(hecuda_cuckoo_table *t) {
    free_table(t);
    return HECUDA_OK;
}

int32_t hecuda_keyword_pir_databases_create(const hecuda_context *h, const hecuda_cuckoo_table *t, int64_t entry_size,
                                            const int32_t *dims, int32_t dim_count, hecuda_pir_database **out) {
    if (!t || !out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const int tables = t->config.table_count();
    for (int i = 0; i < tables; ++i) out[i] = nullptr;
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (h != t->owner) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: the table was built on another context");
    if (!t->config.multiple_tables) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCuckooConfig: keyword PIR needs multipleTables");
    unsigned char *d_bytes = nullptr;
    cudaError_t e = cudaMalloc(&d_bytes, std::max<uint64_t>(t->offsets.back(), 1));
    if (e == cudaSuccess) e = launch_bucket_serialize(t, d_bytes);
    if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) {
        cudaFree(d_bytes);
        return cuda_fail(e, "keyword pir bucket serialization");
    }
    rc = pir_databases_from_device_entries(h, d_bytes, t->offsets.data(), t->d_offsets, t->buckets_per_table, tables,
                                           entry_size, dims, dim_count, out);
    cudaFree(d_bytes);
    return rc;
}

}  // extern "C"
