// capi_internal.hpp -- state behind the opaque handles of include/hecuda.h and the device-side op bodies
// (enqueue-only "chunk" functions) shared by capi.cu and pir.cu.
#pragma once
#include "../../include/hecuda.h"

#include <cuda_runtime.h>

#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "context.hpp"
#include "kernels.cuh"

namespace hecuda {
namespace api {

int32_t fail(int32_t code, const std::string &msg);      // records the thread's last error, returns `code`
int32_t cuda_fail(cudaError_t e, const char *what);
const char *last_error_cstr();

#define CK(expr)                                                          \
    do {                                                                  \
        cudaError_t e_ = (expr);                                          \
        if (e_ != cudaSuccess) return ::hecuda::api::cuda_fail(e_, #expr); \
    } while (0)

// Setup-time uploads (keys, databases, per-call operands staged outside a workspace).  cudaMemcpy from pageable host
// memory may return once the data is staged, before the DMA has reached the device, and cudaMemset on device memory is
// asynchronous; the consumers run on cudaStreamNonBlocking workspace streams or caller streams that do not
// synchronise with the legacy default stream.  So every such upload waits for the legacy stream before the pointer is
// published or used on another stream.
inline cudaError_t upload(void *dst, const void *src, size_t bytes) {
    cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
    return e != cudaSuccess ? e : cudaStreamSynchronize(cudaStreamLegacy);
}
inline cudaError_t fill(void *dst, int value, size_t bytes) {
    cudaError_t e = cudaMemset(dst, value, bytes);
    return e != cudaSuccess ? e : cudaStreamSynchronize(cudaStreamLegacy);
}

// A device buffer that grows on demand and never shrinks.
struct GrowBuffer {
    u64 *p = nullptr;
    size_t cap = 0;  // words
    cudaError_t reserve(size_t words) {
        if (cap >= words) return cudaSuccess;
        if (p) {
            cudaError_t e = cudaFree(p);
            if (e != cudaSuccess) return e;
            p = nullptr;
            cap = 0;
        }
        cudaError_t e = cudaMalloc(&p, words * sizeof(u64));
        if (e == cudaSuccess) cap = words;
        return e;
    }
};

// A stream and what one in-flight stage of the host pipeline (capi.cu) stages through it.
struct Workspace {
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    GrowBuffer scratch, in, out;  // kernel scratch, staged inputs (back to back), staged output
    GrowBuffer in32, out32;       // the uint32 images of `in` and `out` when the host buffers hold uint32 words
    void release() {
        for (GrowBuffer *b : {&scratch, &in, &out, &in32, &out32})
            if (b->p) cudaFree(b->p);
        if (owns_stream && stream) cudaStreamDestroy(stream);
    }
};


}  // namespace api
}  // namespace hecuda

namespace hecuda {
namespace api {
struct PirGraph;  // captured MulPir response pipeline (pir.cu)
void pir_graphs_purge(hecuda_context *h, const void *evk_or_database);  // drop the graphs that reference a handle (nullptr: all)
void context_registered(const hecuda_context *h, bool alive);            // contexts whose graph cache may be touched
}  // namespace api
}  // namespace hecuda

struct hecuda_context {
    hecuda::Context *ctx = nullptr;
    std::vector<hecuda::api::PirGraph *> pir_graphs;  // guarded by mu
    // device copies of MulPir expansion plans by (query ciphertexts, outputs), uploaded once; guarded by mu
    std::map<std::pair<int64_t, int64_t>, void *> expand_steps;
    int64_t chunk = 32;  // ciphertexts per pipeline stage
    std::mutex mu;
    std::vector<hecuda::api::Workspace *> free_ws;  // pooled workspaces (each with its own stream)
    hecuda::api::Workspace *acquire() {
        std::lock_guard<std::mutex> g(mu);
        if (!free_ws.empty()) {
            hecuda::api::Workspace *w = free_ws.back();
            free_ws.pop_back();
            return w;
        }
        hecuda::api::Workspace *w = new (std::nothrow) hecuda::api::Workspace();
        if (!w) return nullptr;
        if (cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) != cudaSuccess) {
            delete w;
            return nullptr;
        }
        w->owns_stream = true;
        return w;
    }
    void release(hecuda::api::Workspace *w) {
        std::lock_guard<std::mutex> g(mu);
        free_ws.push_back(w);
    }
};

struct hecuda_evk {
    const hecuda_context *owner = nullptr;
    unsigned long long version = 0;  // bumped whenever key material changes (captured graphs bake the key pointers in)
    hecuda::u64 *d_relin = nullptr;  // L x 2 x K x N, Eval
    size_t words = 0;
    bool loaded = false;
    std::map<uint32_t, hecuda::u64 *> galois;  // GaloisKey.keys: element -> key-switch key (Keys.swift:150-163), same layout
    std::vector<hecuda::u64 *> retired;        // replaced Galois keys, kept until destroy (in-flight kernels may read them)
    // hecuda_evk_create_serialized(_many): one allocation holding d_relin and the loaded Galois keys.  Pointers into it
    // are freed with it, never on their own; d_relin, galois and retired entries outside it are separate allocations.
    hecuda::u64 *d_block = nullptr;
    size_t block_words = 0;
    bool owns(const hecuda::u64 *p) const { return p && !(p >= d_block && p < d_block + block_words); }
    std::mutex mu;
};

namespace hecuda {
namespace api {

struct WsGuard {
    hecuda_context *h;
    Workspace *w;
    WsGuard(const hecuda_context *hc) : h(const_cast<hecuda_context *>(hc)), w(h->acquire()) {}
    ~WsGuard() {
        if (w) h->release(w);
    }
};

int32_t check_ctx(const hecuda_context *h);

// ---- the staging of the processed-database pipelines (saving and loading PIR and PNNS databases)
// A caller's buffer that is pinned from its first to its last byte (hecuda_host_alloc, hecuda_host_register) is copied
// from directly; a pageable one goes through pinned staging.
inline bool host_pinned(const void *p, size_t bytes) {
    for (const char *at : {(const char *)p, (const char *)p + bytes - 1}) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, at) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        if (a.type != cudaMemoryTypeHost) return false;
    }
    return true;
}

// The pipeline's buffers: two pooled workspaces, each a stream and a device staging buffer (its staged-input buffer,
// which stays with the workspace for later calls), and for a pageable caller buffer a pinned buffer per stream with the
// event after which it may be reused.  The streams are synchronized before this is destroyed.
struct DbStaging {
    WsGuard g0, g1;
    cudaStream_t stream[2];
    unsigned char *dev[2] = {nullptr, nullptr}, *host[2] = {nullptr, nullptr};
    cudaEvent_t copied[2] = {nullptr, nullptr};
    explicit DbStaging(const hecuda_context *h) : g0(h), g1(h) {
        stream[0] = g0.w ? g0.w->stream : nullptr;
        stream[1] = g1.w ? g1.w->stream : nullptr;
    }
    cudaError_t init(size_t bytes, bool pageable) {
        if (!g0.w || !g1.w) return cudaErrorMemoryAllocation;
        Workspace *w[2] = {g0.w, g1.w};
        for (int b = 0; b < 2; ++b) {
            cudaError_t e = w[b]->in.reserve((bytes + sizeof(u64) - 1) / sizeof(u64));
            dev[b] = (unsigned char *)w[b]->in.p;
            if (e == cudaSuccess && pageable) e = cudaHostAlloc(&host[b], bytes, cudaHostAllocDefault);
            if (e == cudaSuccess && pageable) e = cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    ~DbStaging() {
        for (int b = 0; b < 2; ++b) {
            if (host[b]) cudaFreeHost(host[b]);
            if (copied[b]) cudaEventDestroy(copied[b]);
        }
    }
};

// Wait for a stream from a host thread: yields the CPU (an event created with cudaEventBlockingSync, one per thread)
// instead of spinning in cudaStreamSynchronize.
cudaError_t wait_stream(cudaStream_t s);
bool make_map(const Context &c, int32_t base, int32_t rows, NttRowMap &map, std::string &err);

// scratch words needed per ciphertext pair / ciphertext / group
size_t multiply_scratch_words(const Context &c);
size_t relinearize_scratch_words(const Context &c, int l);
size_t galois_scratch_words(const Context &c, int l);
size_t inner_product_scratch_words(const Context &c, int64_t pairs);

cudaError_t multiply_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, u64 *out, int64_t items,
                           cudaStream_t s);
// keys: one key per client (launch_ks_mac) in place of `key`
cudaError_t keyswitch_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *target, int64_t target_stride,
                            int l, const u64 *base, int64_t base_stride, int base_mask, u64 *out, int64_t items,
                            cudaStream_t s, const KsKeyTable *keys = nullptr);
cudaError_t relinearize_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct3, int l, u64 *out,
                              int64_t items, cudaStream_t s, const KsKeyTable *keys = nullptr);
cudaError_t apply_galois_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct, int l, unsigned element,
                               u64 *out, int64_t items, cudaStream_t s, const KsKeyTable *keys = nullptr);
// with at.tag: poly0 and seeds read in place from the bytes at d_poly0 (at.tag / at.seed, drbg.cu)
cudaError_t expand_seeded_device(const Context &c, int l, const unsigned char *d_poly0, const unsigned char *d_seeds, u64 *d_out,
                                 int64_t batch, cudaStream_t s, const PolyLayout &at = PolyLayout{});
// Seeded key-switching ciphertexts (K = L + 1 rows, Eval) in two steps: drbg_chains over their seeds with
// key_segments(c) segments each, then ciphertexts [first, first + count) from those chains: d_poly0 holds their
// count x byteCount(K rows) bytes, and ciphertext i's 2 x K x N words go to d_dst[i] (a device table of pointers into
// evaluation keys).  With layout.tag, ciphertext first + i's poly0 is at d_poly0 + layout.tag[layout.first + i] -
// layout.base instead.
int key_segments(const Context &c);
cudaError_t expand_key_ciphertexts(const Context &c, const unsigned int *d_rk, const u64 *d_ctr, int64_t first, int64_t count,
                                   const unsigned char *d_poly0, u64 *const *d_dst, cudaStream_t s,
                                   const PolyLayout &layout = PolyLayout{});
// NistAes128Ctr streams (drbg.cu): the AES tables, then for every 32-byte seed the round keys (segments x 44 words) and
// counters V (segments x 2 words) of its first `segments` 4096-byte segments; free_chains zeroizes the round keys.
// Seed b is at d_seeds + 32 b, or at d_seeds + d_seed_at[b] (a device table) when one is given.
cudaError_t drbg_chains(const unsigned char *d_seeds, int segments, int64_t batch, unsigned int **d_rk, u64 **d_ctr,
                        cudaStream_t s, const long long *d_seed_at = nullptr);
void free_chains(unsigned int *d_rk, u64 *d_ctr, int segments, int64_t batch, cudaStream_t s);
// drbg_chains in two steps: the AES tables (synchronises s), then the chains alone (stream-ordered and graph-capturable
// once the tables are on the device)
cudaError_t drbg_upload_tables(cudaStream_t s);
cudaError_t drbg_chains_uploaded(const unsigned char *d_seeds, int segments, int64_t batch, unsigned int **d_rk, u64 **d_ctr,
                                 cudaStream_t s, const long long *d_seed_at = nullptr);
cudaError_t drbg_tables(const unsigned char **sbox, const unsigned int **te0);
// PolyRq.random mod p of `polys` degree-n polynomials from the one stream of the 32-byte d_seed (coefficient k of
// polynomial j is the stream's (jN + k)-th 128-bit word mod p), stored as sigma(a) = a(x^-1) (simple_pir.cuh)
cudaError_t random_sigma_polys_device(const unsigned char *d_seed, u64 p, int64_t n, int64_t polys, u64 *d_out,
                                      cudaStream_t s);
// the same polynomials as a itself (SimplePirContext.generateAPolynomials for the client)
cudaError_t random_polys_one_modulus_device(const unsigned char *d_seed, u64 p, int64_t n, int64_t polys, bool sigma,
                                            u64 *d_out, cudaStream_t s);
// SimplePirParameters' checks and derived sizes (simple_pir.cu): DB' is m x k (columnSize x databaseColumns), an entry
// is entry_scalars coefficients, p = nttFriendlyMod
int32_t simple_pir_derive(const hecuda_simple_pir_params *params, int64_t &m, int64_t &k, int64_t &entry_scalars, u64 &p);
cudaError_t inner_product_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, int64_t pairs, u64 *out,
                                int64_t groups, cudaStream_t s);
// `tables` MulPir databases from entry bytes already on the device (pir.cu; used by keyword_pir.cu)
int32_t pir_databases_from_device_entries(const hecuda_context *h, const unsigned char *d_entries, const uint64_t *h_offsets,
                                          const uint64_t *d_offsets, int64_t per_table, int tables, int64_t entry_size,
                                          const int32_t *dims, int32_t dim_count, hecuda_pir_database **out);

// Bfv.encrypt of `batch` plaintexts already on the device (client.cu): d_sk L x N (Eval), d_pt batch x N (< t), seeds
// batch x 32 each -> d_c0 batch x L x N (Coeff) and d_c1 = d_c0 + batch x L x N (Coeff with c1_coeff, else Eval)
cudaError_t encrypt_plaintexts_device(const Context &c, const u64 *d_sk, const u64 *d_pt, const unsigned char *d_a_seeds,
                                      const unsigned char *d_e_seeds, u64 *d_c0, u64 *d_c1, bool c1_coeff, int64_t batch,
                                      cudaStream_t s);
// Bfv.decryptCoeff of `items` ciphertexts of polys x l x N on the device (decrypt.cu) -> out items x N (< t); scratch:
// decrypt_scratch_words per item
size_t decrypt_scratch_words(const Context &c, int polys, int l);
cudaError_t decrypt_device(const Context &c, const u64 *d_sk, const u64 *d_ct, int polys, int l, u64 *scratch, u64 *out,
                           int64_t items, cudaStream_t s);
// The host-side refusals of a float front end (pnns_client.cu): a null or non-finite vector value, a negative scaling
// factor, or one whose scaled values cannot fit the plaintext map (Int64 with `reduce`, else the centred range mod t).
// scan: look for non-finite values on the host (else the device's normalisation flags them)
int32_t check_float_vectors(const float *vectors, int64_t rows, int64_t cols, int64_t scaling_factor, u64 t, bool reduce,
                            bool scan);

}  // namespace api
}  // namespace hecuda
