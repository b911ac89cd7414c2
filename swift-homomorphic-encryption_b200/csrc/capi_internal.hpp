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

// Scratch for one in-flight chunk.  Grows on demand, never shrinks.
struct Workspace {
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    u64 *buf[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    size_t cap[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    cudaError_t reserve(int i, size_t words) {
        if (cap[i] >= words) return cudaSuccess;
        if (buf[i]) {
            cudaError_t e = cudaFree(buf[i]);
            if (e != cudaSuccess) return e;
            buf[i] = nullptr;
            cap[i] = 0;
        }
        cudaError_t e = cudaMalloc(&buf[i], words * sizeof(u64));
        if (e == cudaSuccess) cap[i] = words;
        return e;
    }
    void release() {
        for (int i = 0; i < 8; ++i)
            if (buf[i]) cudaFree(buf[i]);
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
cudaError_t keyswitch_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *target, int64_t target_stride,
                            int l, const u64 *base, int64_t base_stride, int base_mask, u64 *out, int64_t items,
                            cudaStream_t s);
cudaError_t relinearize_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct3, int l, u64 *out,
                              int64_t items, cudaStream_t s);
cudaError_t apply_galois_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct, int l, unsigned element,
                               u64 *out, int64_t items, cudaStream_t s);
cudaError_t expand_seeded_device(const Context &c, int l, const unsigned char *d_poly0, const unsigned char *d_seeds, u64 *d_out,
                                 int64_t batch, cudaStream_t s);
cudaError_t inner_product_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, int64_t pairs, u64 *out,
                                int64_t groups, cudaStream_t s);

}  // namespace api
}  // namespace hecuda
