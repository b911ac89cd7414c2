// capi.cu -- the C ABI declared in include/hecuda.h.  No torch types, no exceptions across the boundary.
//
// Host-pointer entry points run a chunked, double-buffered pipeline (two workspaces on two streams) so that the
// H2D copy of chunk k+1, the kernels of chunk k and the D2H copy of chunk k-1 overlap when the caller's buffers are
// pinned.  Device-pointer entry points enqueue on the caller's stream and do not synchronize.
#include "../../include/hecuda.h"

#include <cuda_runtime.h>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "capi_internal.hpp"

namespace hecuda {
std::atomic<unsigned long long> g_kernel_launches{0};
}

using namespace hecuda;

namespace hecuda {
namespace api {

static thread_local std::string tl_error;

int32_t fail(int32_t code, const std::string &msg) {
    tl_error = msg;
    return code;
}
int32_t cuda_fail(cudaError_t e, const char *what) {
    return fail(HECUDA_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
const char *last_error_cstr() { return tl_error.c_str(); }

}  // namespace api
}  // namespace hecuda

using namespace hecuda::api;

namespace hecuda {
namespace api {

cudaError_t wait_stream(cudaStream_t s) {
    // Yield the CPU while waiting (an event created with cudaEventBlockingSync).  Spinning in cudaStreamSynchronize
    // burns a core per waiting thread; with many serving threads inside a CPU-quota'd container the spinners get
    // throttled and throughput collapses and swings from run to run.
    thread_local cudaEvent_t event = nullptr;
    thread_local int event_device = -1;
    int device = 0;
    cudaError_t e = cudaGetDevice(&device);
    if (e != cudaSuccess) return e;
    if (!event || event_device != device) {
        if ((e = cudaEventCreateWithFlags(&event, cudaEventBlockingSync | cudaEventDisableTiming)) != cudaSuccess) return e;
        event_device = device;
    }
    if ((e = cudaEventRecord(event, s)) != cudaSuccess) return e;
    return cudaEventSynchronize(event);
}

int32_t check_ctx(const hecuda_context *h) {
    if (!h || !h->ctx) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: null context");
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device available");
    if (dev != h->ctx->device) {
        cudaError_t e = cudaSetDevice(h->ctx->device);
        if (e != cudaSuccess) return cuda_fail(e, "cudaSetDevice");
    }
    return HECUDA_OK;
}

bool make_map(const Context &c, int32_t base, int32_t rows, NttRowMap &map, std::string &err) {
    switch (base) {
        case HECUDA_BASE_Q:
            if (rows < 1 || rows > c.L) { err = "invalidPolyContext: row_count must be in [1, L] for BASE_Q"; return false; }
            map = c.map_q(rows);
            return true;
        case HECUDA_BASE_Q_BSK:
            if (rows != 2 * c.L + 1) { err = "invalidPolyContext: BASE_Q_BSK needs 2L+1 rows"; return false; }
            map = c.map_qbsk();
            return true;
        case HECUDA_BASE_Q_AUX:
            if (rows != 2 * c.L + 1) { err = "invalidPolyContext: BASE_Q_AUX needs 2L+1 rows"; return false; }
            map = c.map_qaux();
            return true;
        case HECUDA_BASE_KEYSWITCH:
            if (!c.has_ks) { err = "invalidPolyContext: these parameters have no key-switching modulus"; return false; }
            if (rows < 2 || rows > c.L + 1) { err = "invalidPolyContext: BASE_KEYSWITCH needs 2..L+1 rows"; return false; }
            map = c.map_ks(rows - 1);
            return true;
        default:
            err = "invalidPolyContext: unknown base";
            return false;
    }
}

// ---------------------------------------------------------------- device-side op bodies (enqueue only)

// scratch words needed per ciphertext pair / ciphertext
size_t multiply_scratch_words(const Context &c) { return (size_t)7 * (2 * c.L + 1) * c.n; }
size_t relinearize_scratch_words(const Context &c, int l) { return (size_t)((l + 1) * l + 2 * (l + 1)) * c.n; }

cudaError_t multiply_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, u64 *out, int64_t items,
                           cudaStream_t s) {
    const int R = 2 * c.L + 1;
    const size_t poly_words = (size_t)R * c.n;
    cudaError_t e;
    u64 *ext = scratch, *ten = scratch + 4 * poly_words * items;
    const NttRowMap map = c.map_qaux();
    // dropExtendedBase: (* t) and the floor's first step ((Q/q_i)^-1 on the Q rows) folded into the inverse NTT
    const bool scaled = floor_takes_scaled_q(c);
    const int inv_scale = scaled ? kScaleTMontFloor : kScaleTMont;
    if (ntt_forward_tensor_supported(c)) {
        // computeBehzPolys + tensor product with the NTT outputs kept on chip (ntt_fast.cu): the lift writes only the
        // auxiliary rows, the kernel reads the Q rows from lhs / rhs
        if ((e = launch_lift(c, lhs, rhs, 2, ext, items, s, false, false)) != cudaSuccess) return e;
        if ((e = launch_ntt_forward_tensor(c, map, lhs, rhs, ext, ten, items, s)) != cudaSuccess) return e;
        if ((e = launch_ntt_inverse(c, map, ten, ten, items * 3 * R, inv_scale, s)) != cudaSuccess) return e;
        return launch_floor(c, ten, out, items * 3, s, false, scaled);
    }
    // computeBehzPolys for both operands: lift + forward NTT      (Bfv+Multiply.swift:51-57)
    if ((e = launch_lift(c, lhs, rhs, 2, ext, items, s)) != cudaSuccess) return e;
    if ((e = launch_ntt_forward(c, map, ext, ext, items * 4 * R, s)) != cudaSuccess) return e;
    // tensor product                                               (Bfv+Multiply.swift:80-82)
    if ((e = launch_tensor(c, ext, ten, items, s)) != cudaSuccess) return e;
    // dropExtendedBase: inverse NTT, floor                          (Bfv+Multiply.swift:31-48)
    if ((e = launch_ntt_inverse(c, map, ten, ten, items * 3 * R, inv_scale, s)) != cudaSuccess) return e;
    return launch_floor(c, ten, out, items * 3, s, false, scaled);
}

// _computeKeySwitchingUpdate (Bfv+Keys.swift:123-208) of `target` (l rows per item, items `target_stride` words apart)
// + the caller's accumulation: out[item][c] = update[c] (+ base[item][c] for the components in base_mask).
cudaError_t keyswitch_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *target, int64_t target_stride,
                            int l, const u64 *base, int64_t base_stride, int base_mask, u64 *out, int64_t items,
                            cudaStream_t s, const KsKeyTable *keys) {
    const size_t dig_words = (size_t)(l + 1) * l * c.n;
    cudaError_t e;
    u64 *dig = scratch, *prod = scratch + dig_words * items;
    // digits: forward NTT that gathers [target row j]_{m_r} straight from the source      (Bfv+Keys.swift:165-179)
    if ((e = launch_ntt_forward(c, c.map_ks_digits(l, target_stride), target, dig, items * (l + 1) * l, s)) != cudaSuccess)
        return e;
    if ((e = launch_ks_mac(c, dig, key, l, prod, items, s, keys)) != cudaSuccess) return e;
    if ((e = launch_ntt_inverse(c, c.map_ks(l), prod, prod, items * 2 * (l + 1), kScaleMont, s)) != cudaSuccess) return e;
    return launch_ks_finish(c, prod, base, base_stride, base_mask, l, out, items, s);
}

// Bfv.relinearize (Bfv.swift:201-219): key-switch poly 2, add the update to polys 0 and 1
cudaError_t relinearize_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct3, int l, u64 *out,
                              int64_t items, cudaStream_t s, const KsKeyTable *keys) {
    const int64_t ct_stride = (int64_t)3 * l * c.n;
    return keyswitch_chunk(c, scratch, key, ct3 + (int64_t)2 * l * c.n, ct_stride, l, ct3, ct_stride, 3, out, items, s, keys);
}

// Bfv.applyGalois (Bfv.swift:174-198): c0' = galois(c0) + update[0], c1' = update[1], update = keyswitch(galois(c1))
size_t galois_scratch_words(const Context &c, int l) { return relinearize_scratch_words(c, l) + (size_t)l * c.n; }
cudaError_t apply_galois_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *ct, int l, unsigned element,
                               u64 *out, int64_t items, cudaStream_t s, const KsKeyTable *keys) {
    const int64_t poly = (int64_t)l * c.n, ct_stride = 2 * poly;
    u64 *perm1 = scratch;                      // items x l x N
    u64 *ks_scratch = scratch + poly * items;
    const NttRowMap map = c.map_q(l);
    cudaError_t e;
    if ((e = launch_galois_coeff(c, map, element, ct, ct_stride, out, ct_stride, items, s)) != cudaSuccess) return e;
    if ((e = launch_galois_coeff(c, map, element, ct + poly, ct_stride, perm1, poly, items, s)) != cudaSuccess) return e;
    return keyswitch_chunk(c, ks_scratch, key, perm1, poly, l, out, ct_stride, 1, out, items, s, keys);
}

// Bfv.innerProduct(_:_:) (Bfv.swift:315-361): sum of the tensor products of `pairs` ciphertext pairs in [Q, Bsk],
// then ONE dropExtendedBase -- instead of `pairs` full multiplies.
cudaError_t inner_product_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, int64_t pairs,
                                       u64 *out, int64_t groups, cudaStream_t s) {
    const int R = 2 * c.L + 1;
    const size_t poly_words = (size_t)R * c.n;
    const int64_t items = groups * pairs;
    u64 *ext = scratch, *ten = scratch + 4 * poly_words * items;
    const NttRowMap map = c.map_qaux();
    cudaError_t e;
    const bool scaled = floor_takes_scaled_q(c);
    if ((e = launch_lift(c, lhs, rhs, 2, ext, items, s)) != cudaSuccess) return e;
    if ((e = launch_ntt_forward(c, map, ext, ext, items * 4 * R, s)) != cudaSuccess) return e;
    if ((e = launch_tensor_sum(c, ext, ten, pairs, groups, s)) != cudaSuccess) return e;
    if ((e = launch_ntt_inverse(c, map, ten, ten, groups * 3 * R, scaled ? kScaleTMontFloor : kScaleTMont, s)) != cudaSuccess)
        return e;
    return launch_floor(c, ten, out, groups * 3, s, false, scaled);
}
size_t inner_product_scratch_words(const Context &c, int64_t pairs) {
    return (size_t)(4 * pairs + 3) * (2 * c.L + 1) * c.n;
}

}  // namespace api
}  // namespace hecuda

namespace {

// The u32 entry points (Bfv<UInt32> contexts) run the same bodies: the calling thread marks its host buffers as uint32
// for the duration of the call and the pipeline widens after the H2D copy / narrows before the D2H copy.
thread_local bool tl_io32 = false;
struct Io32Scope {
    Io32Scope() { tl_io32 = true; }
    ~Io32Scope() { tl_io32 = false; }
};

// Generic double-buffered host pipeline: for each chunk, copy inputs in, run `body`, copy outputs out.
struct HostIo {
    const u64 *src;  // host
    size_t words_per_item;
};
template <class Body>
int32_t host_pipeline(const hecuda_context *h, int64_t batch, int64_t chunk_hint, size_t scratch_words_per_item,
                      const std::vector<HostIo> &inputs, u64 *host_out, size_t out_words_per_item, Body body) {
    if (batch == 0) return HECUDA_OK;
    // `depth` stages in flight, each on its own stream: H2D of stage k+1.., kernels of stage k, D2H of stage k-1
    static const int depth = [] {
        const char *env = std::getenv("HECUDA_PIPELINE_DEPTH");
        const int d = env ? std::atoi(env) : 3;
        return d < 1 ? 1 : (d > 8 ? 8 : d);
    }();
    static const int64_t min_stages = [] {
        const char *env = std::getenv("HECUDA_PIPELINE_STAGES");
        const long long v = env ? std::atoll(env) : 16;
        return (int64_t)(v < 1 ? 1 : v);
    }();
    std::vector<std::unique_ptr<WsGuard>> guards;
    std::vector<Workspace *> ws;
    for (int i = 0; i < depth; ++i) {
        guards.emplace_back(new WsGuard(h));
        if (!guards.back()->w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
        ws.push_back(guards.back()->w);
    }
    int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(chunk_hint, batch));
    if (batch >= 64) chunk = std::min<int64_t>(chunk, std::max<int64_t>(16, (batch + min_stages - 1) / min_stages));
    // On any early return, earlier stages may still have copies into / out of the caller's buffers in flight on the
    // other streams: wait for all of them so the caller may free or reuse its buffers as soon as it sees the error.
    struct DrainOnExit {
        std::vector<Workspace *> &ws;
        ~DrainOnExit() {
            for (Workspace *w : ws) wait_stream(w->stream);
        }
    } drain{ws};
    int k = 0;
    for (int64_t done = 0; done < batch; done += chunk, ++k) {
        Workspace &w = *ws[k % depth];
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        // Work on one workspace is ordered by its stream; buffers only ever grow (first `depth` iterations).
        // slot 0 = kernel scratch, slot 4 = staged inputs (back to back), slot 5 = staged output
        size_t in_words = 0;
        for (const HostIo &io : inputs) in_words += io.words_per_item * (size_t)items;
        const bool io32 = tl_io32;
        const size_t out_words = out_words_per_item * (size_t)items;
        CK(w.reserve(0, scratch_words_per_item * (size_t)items));
        CK(w.reserve(4, in_words));
        CK(w.reserve(5, out_words));
        if (io32) {  // slots 6 / 7: the uint32 images (each input starts on a 16-byte boundary)
            CK(w.reserve(6, in_words / 2 + inputs.size() * 2 + 2));
            CK(w.reserve(7, out_words / 2 + 2));
        }
        std::vector<const u64 *> d_in;
        size_t off = 0, off32 = 0;
        for (const HostIo &io : inputs) {
            const size_t words = io.words_per_item * (size_t)items;
            if (io32) {
                u32 *raw = reinterpret_cast<u32 *>(w.buf[6]) + off32;
                CK(cudaMemcpyAsync(raw, reinterpret_cast<const u32 *>(io.src) + io.words_per_item * (size_t)done,
                                   words * sizeof(u32), cudaMemcpyHostToDevice, w.stream));
                CK(launch_widen(raw, w.buf[4] + off, (int64_t)words, w.stream));
                off32 += (words + 3) & ~(size_t)3;
            } else {
                CK(cudaMemcpyAsync(w.buf[4] + off, io.src + io.words_per_item * (size_t)done, words * sizeof(u64),
                                   cudaMemcpyHostToDevice, w.stream));
            }
            d_in.push_back(w.buf[4] + off);
            off += words;
        }
        cudaError_t e = body(w, d_in, w.buf[5], items);
        if (e != cudaSuccess) return cuda_fail(e, "kernel launch");
        if (io32) {
            CK(launch_narrow(w.buf[5], reinterpret_cast<u32 *>(w.buf[7]), (int64_t)out_words, w.stream));
            CK(cudaMemcpyAsync(reinterpret_cast<u32 *>(host_out) + out_words_per_item * (size_t)done, w.buf[7],
                               out_words * sizeof(u32), cudaMemcpyDeviceToHost, w.stream));
        } else {
            CK(cudaMemcpyAsync(host_out + out_words_per_item * (size_t)done, w.buf[5], out_words * sizeof(u64),
                               cudaMemcpyDeviceToHost, w.stream));
        }
    }
    for (Workspace *w : ws) CK(wait_stream(w->stream));
    return HECUDA_OK;
}

}  // namespace

// ====================================================================================================== C ABI

extern "C" {

int32_t hecuda_version(void) { return 100; }
const char *hecuda_last_error(void) { return last_error_cstr(); }

int32_t hecuda_device_count(int32_t *count) {
    if (!count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null count");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        *count = 0;
        return fail(HECUDA_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e));
    }
    *count = n;
    return HECUDA_OK;
}
int32_t hecuda_set_device(int32_t device) {
    CK(cudaSetDevice(device));
    return HECUDA_OK;
}

// NUMA placement of the host side of one GPU: pin the calling thread (threads it creates later inherit the mask) to the
// CPUs local to the GPU's PCIe root and prefer that node for page allocations, so that pinned staging buffers
// allocated afterwards (hecuda_host_alloc) and the copies out of them do not cross the socket interconnect.
int32_t hecuda_bind_host_to_device(int32_t device, int32_t *numa_node, int32_t *cpu_count) {
    if (numa_node) *numa_node = -1;
    if (cpu_count) *cpu_count = 0;
    char bus[32] = {0};
    CK(cudaDeviceGetPCIBusId(bus, sizeof(bus), device));
    for (char *c = bus; *c; ++c) *c = (char)std::tolower((unsigned char)*c);
    const std::string dir = std::string("/sys/bus/pci/devices/") + bus + "/";
    int node = -1;
    if (FILE *f = std::fopen((dir + "numa_node").c_str(), "r")) {
        if (std::fscanf(f, "%d", &node) != 1) node = -1;
        std::fclose(f);
    }
    char list[4096] = {0};
    if (FILE *f = std::fopen((dir + "local_cpulist").c_str(), "r")) {
        if (!std::fgets(list, sizeof(list), f)) list[0] = 0;
        std::fclose(f);
    }
    cpu_set_t current, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof(current), &current) != 0) return HECUDA_OK;  // nothing to intersect with: leave as is
    int picked = 0;
    char *save = nullptr;
    for (char *tok = strtok_r(list, ",\n", &save); tok; tok = strtok_r(nullptr, ",\n", &save)) {
        int lo = 0, hi = 0;
        const int fields = std::sscanf(tok, "%d-%d", &lo, &hi);
        if (fields < 1) continue;
        if (fields == 1) hi = lo;
        for (int c = lo; c <= hi && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET(c, &current)) {
                CPU_SET(c, &want);
                ++picked;
            }
    }
    if (picked > 0) sched_setaffinity(0, sizeof(want), &want);
    if (node >= 0 && node < 64) {  // MPOL_PREFERRED: fall back to other nodes rather than fail when the node is full
        unsigned long mask = 1ul << node;
        syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, sizeof(mask) * 8);
    }
    if (numa_node) *numa_node = node;
    if (cpu_count) *cpu_count = picked;
    return HECUDA_OK;
}

int32_t hecuda_host_alloc(void **ptr, uint64_t bytes) {
    if (!ptr) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null ptr");
    CK(cudaHostAlloc(ptr, bytes, cudaHostAllocDefault));
    return HECUDA_OK;
}
int32_t hecuda_host_free(void *ptr) {
    CK(cudaFreeHost(ptr));
    return HECUDA_OK;
}
int32_t hecuda_host_register(void *ptr, uint64_t bytes) {
    CK(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
    return HECUDA_OK;
}
int32_t hecuda_host_unregister(void *ptr) {
    CK(cudaHostUnregister(ptr));
    return HECUDA_OK;
}

static int32_t context_create(int64_t poly_degree, const uint64_t *coefficient_moduli, int32_t moduli_count,
                              uint64_t plaintext_modulus, int word_bits, hecuda_context **out);
int32_t hecuda_context_create(int64_t poly_degree, const uint64_t *coefficient_moduli, int32_t moduli_count,
                              uint64_t plaintext_modulus, hecuda_context **out) {
    return context_create(poly_degree, coefficient_moduli, moduli_count, plaintext_modulus, 64, out);
}
int32_t hecuda_context_create_u32(int64_t poly_degree, const uint32_t *coefficient_moduli, int32_t moduli_count,
                                  uint32_t plaintext_modulus, hecuda_context **out) {
    if (!coefficient_moduli || moduli_count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    std::vector<uint64_t> wide(coefficient_moduli, coefficient_moduli + moduli_count);
    return context_create(poly_degree, wide.data(), moduli_count, plaintext_modulus, 32, out);
}
int32_t hecuda_context_word_bits(const hecuda_context *h, int32_t *bits) {
    if (!h || !bits) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *bits = h->ctx->word_bits;
    return HECUDA_OK;
}
static int32_t context_create(int64_t poly_degree, const uint64_t *coefficient_moduli, int32_t moduli_count,
                              uint64_t plaintext_modulus, int word_bits, hecuda_context **out) {
    if (!out || !coefficient_moduli) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    std::string err;
    Context *c = Context::create(poly_degree, (const u64 *)coefficient_moduli, moduli_count, plaintext_modulus, err, word_bits);
    if (!c) {
        const bool unsupported = err.rfind("unsupported", 0) == 0;
        return fail(unsupported ? HECUDA_ERR_UNSUPPORTED : HECUDA_ERR_INVALID_ARGUMENT, err);
    }
    hecuda_context *h = new (std::nothrow) hecuda_context();
    if (!h) {
        delete c;
        return fail(HECUDA_ERR_CUDA, "out of host memory");
    }
    h->ctx = c;
    {   // keep stream-ordered scratch cached in the default pool instead of returning it to the OS at every sync
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, c->device) == cudaSuccess) {
            unsigned long long threshold = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
        }
    }
    // pipeline stage size: keep one stage's intermediates (7 R N words per ciphertext pair) near the L2 size
    // Every kernel on this path is instruction-issue bound, not HBM bound (DESIGN.md), so large launches that
    // amortise wave tails beat L2-resident small ones: size a stage to ~2 GB of scratch.
    const size_t per_item = (size_t)7 * (2 * c->L + 1) * c->n * sizeof(u64);
    int64_t chunk = (int64_t)((size_t)2048 * 1024 * 1024 / per_item);
    if (const char *env = std::getenv("HECUDA_CHUNK")) chunk = std::atoll(env);
    h->chunk = std::max<int64_t>(1, std::min<int64_t>(chunk, 4096));
    context_registered(h, true);
    *out = h;
    return HECUDA_OK;
}

int32_t hecuda_context_destroy(hecuda_context *h) {
    if (!h) return HECUDA_OK;
    if (h->ctx) cudaSetDevice(h->ctx->device);
    cudaDeviceSynchronize();
    pir_graphs_purge(h, nullptr);
    context_registered(h, false);
    for (auto &kv : h->expand_steps) cudaFree(kv.second);
    for (Workspace *w : h->free_ws) {
        w->release();
        delete w;
    }
    delete h->ctx;
    delete h;
    return HECUDA_OK;
}

int32_t hecuda_context_ciphertext_moduli_count(const hecuda_context *h, int32_t *count) {
    if (!h || !count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *count = h->ctx->L;
    return HECUDA_OK;
}
int32_t hecuda_context_bsk_moduli(const hecuda_context *h, uint64_t *out, int32_t capacity, int32_t *count) {
    if (!h || !count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *count = (int32_t)h->ctx->bsk.size();
    if (out) {
        if (capacity < *count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity too small");
        std::memcpy(out, h->ctx->bsk.data(), sizeof(u64) * h->ctx->bsk.size());
    }
    return HECUDA_OK;
}
int32_t hecuda_context_aux_moduli(const hecuda_context *h, uint64_t *out, int32_t capacity, int32_t *count) {
    if (!h || !count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *count = (int32_t)h->ctx->aux.size();
    if (out) {
        if (capacity < *count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity too small");
        std::memcpy(out, h->ctx->aux.data(), sizeof(u64) * h->ctx->aux.size());
    }
    return HECUDA_OK;
}
int32_t hecuda_context_root_tables(const hecuda_context *h, uint64_t modulus, uint64_t *roots, uint64_t *inverse_roots) {
    if (!h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null context");
    const int s = h->ctx->find_slot(modulus);
    if (s < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidNttModulus: modulus is not part of this context");
    if (roots) std::memcpy(roots, h->ctx->slots[s].roots.data(), sizeof(u64) * h->ctx->n);
    if (inverse_roots) std::memcpy(inverse_roots, h->ctx->slots[s].inv_roots.data(), sizeof(u64) * h->ctx->n);
    return HECUDA_OK;
}

// ---------------------------------------------------------------- NTT

static int32_t ntt_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys,
                          void *stream, bool inverse) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (!data && polys)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    cudaError_t e = inverse ? launch_ntt_inverse(*h->ctx, map, (u64 *)data, (u64 *)data, polys * rows, kScalePlain,
                                                 (cudaStream_t)stream)
                            : launch_ntt_forward(*h->ctx, map, (u64 *)data, (u64 *)data, polys * rows,
                                                 (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "ntt launch");
    return HECUDA_OK;
}
int32_t hecuda_ntt_forward_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys,
                                  void *stream) {
    return ntt_device(h, base, data, rows, polys, stream, false);
}
int32_t hecuda_ntt_inverse_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys,
                                  void *stream) {
    return ntt_device(h, base, data, rows, polys, stream, true);
}

static int32_t ntt_host(const hecuda_context *h, const NttRowMap &map, uint64_t *data, size_t words_per_item,
                        int64_t items, int64_t rows_per_item, bool inverse) {
    const Context &c = *h->ctx;
    std::vector<HostIo> in = {{(const u64 *)data, words_per_item}};
    // NTT items are single polynomials: stage ~32 MB per pipeline step
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / std::max<size_t>(1, words_per_item)));
    return host_pipeline(h, items, chunk, 0, in, (u64 *)data, words_per_item,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t n_items) {
                             return inverse ? launch_ntt_inverse(c, map, d_in[0], d_out, n_items * rows_per_item, kScalePlain,
                                                                 w.stream)
                                            : launch_ntt_forward(c, map, d_in[0], d_out, n_items * rows_per_item,
                                                                 w.stream);
                         });
}
int32_t hecuda_ntt_forward(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (!data && polys)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    return ntt_host(h, map, data, (size_t)rows * h->ctx->n, polys, rows, false);
}
int32_t hecuda_ntt_inverse(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (!data && polys)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    return ntt_host(h, map, data, (size_t)rows * h->ctx->n, polys, rows, true);
}
// Stage-level BEHZ entry points over the reference's [Q, Bsk] (RnsTool.swift:324-331, 453-456), Coeff format.
int32_t hecuda_rnstool_lift_q_to_qbsk(const hecuda_context *h, const uint64_t *polys, uint64_t *out, int64_t count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (count < 0 || ((!polys || !out) && count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid buffers / poly_count");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)c.L * c.n, out_words = (size_t)(2 * c.L + 1) * c.n;
    std::vector<HostIo> in = {{(const u64 *)polys, in_words}};
    return host_pipeline(h, count, std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / out_words)), 0, in, (u64 *)out, out_words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t n_items) {
                             return launch_lift(c, d_in[0], nullptr, 1, d_out, n_items, w.stream, /*reference_base=*/true);
                         });
}
int32_t hecuda_rnstool_floor_qbsk_to_q(const hecuda_context *h, const uint64_t *polys, uint64_t *out, int64_t count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (count < 0 || ((!polys || !out) && count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid buffers / poly_count");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)(2 * c.L + 1) * c.n, out_words = (size_t)c.L * c.n;
    std::vector<HostIo> in = {{(const u64 *)polys, in_words}};
    return host_pipeline(h, count, std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / in_words)), 0, in, (u64 *)out, out_words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t n_items) {
                             return launch_floor(c, d_in[0], d_out, n_items, w.stream, /*reference_base=*/true);
                         });
}

static int32_t ntt_rows_host(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows, bool inverse) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (rows < 0 || (!data && rows)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / row_count");
    const int s = h->ctx->find_slot(modulus);
    if (s < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modulus is not part of this context");
    return ntt_host(h, h->ctx->map_single(s), data, (size_t)h->ctx->n, rows, 1, inverse);
}
int32_t hecuda_ntt_forward_rows(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows) {
    return ntt_rows_host(h, modulus, data, rows, false);
}
int32_t hecuda_ntt_inverse_rows(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows) {
    return ntt_rows_host(h, modulus, data, rows, true);
}

// ---------------------------------------------------------------- multiply

int32_t hecuda_bfv_multiply_device(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                   int64_t batch, void *stream) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (batch < 0 || (batch && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    if (batch == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n, out_words = (size_t)3 * c.L * c.n;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, batch));
    cudaStream_t s = (cudaStream_t)stream;
    u64 *scratch = nullptr;  // stream-ordered scratch: no host synchronization, graph-capturable
    CK(cudaMallocAsync(&scratch, multiply_scratch_words(c) * (size_t)chunk * sizeof(u64), s));
    for (int64_t done = 0; done < batch; done += chunk) {
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        cudaError_t e = multiply_chunk(c, scratch, (const u64 *)lhs + in_words * done, (const u64 *)rhs + in_words * done,
                                       (u64 *)out + out_words * done, items, s);
        if (e != cudaSuccess) {
            cudaFreeAsync(scratch, s);
            return cuda_fail(e, "multiply");
        }
    }
    CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}

int32_t hecuda_bfv_multiply(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                            int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (batch < 0 || (batch && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n, out_words = (size_t)3 * c.L * c.n;
    std::vector<HostIo> in = {{(const u64 *)lhs, in_words}, {(const u64 *)rhs, in_words}};
    return host_pipeline(h, batch, h->chunk, multiply_scratch_words(c), in, (u64 *)out, out_words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return multiply_chunk(c, w.buf[0], d_in[0], d_in[1], d_out, items, w.stream);
                         });
}

// ---------------------------------------------------------------- evaluation key

int32_t hecuda_evk_create_empty(const hecuda_context *h, hecuda_evk **out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *h->ctx;
    if (!c.has_ks)  // Context.supportsEvaluationKey == false with a single coefficient modulus (Context.swift:102-107)
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: a single coefficient modulus leaves no key-switching modulus");
    hecuda_evk *k = new (std::nothrow) hecuda_evk();
    if (!k) return fail(HECUDA_ERR_CUDA, "out of host memory");
    k->owner = h;
    k->words = (size_t)c.L * 2 * (c.L + 1) * c.n;
    cudaError_t e = cudaMalloc(&k->d_relin, k->words * sizeof(u64));
    if (e != cudaSuccess) {
        delete k;
        return cuda_fail(e, "cudaMalloc(evk)");
    }
    *out = k;
    return HECUDA_OK;
}
int32_t hecuda_evk_create(const hecuda_context *h, const uint64_t *relin_key, hecuda_evk **out) {
    if (!relin_key) return fail(HECUDA_ERR_MISSING_KEY, "missingRelinearizationKey");
    int32_t rc = hecuda_evk_create_empty(h, out);
    if (rc) return rc;
    cudaError_t e = upload((*out)->d_relin, relin_key, (*out)->words * sizeof(u64));
    if (e != cudaSuccess) {
        hecuda_evk_destroy(*out);
        *out = nullptr;
        return cuda_fail(e, "cudaMemcpy(evk)");
    }
    (*out)->loaded = true;
    return HECUDA_OK;
}
int32_t hecuda_evk_destroy(hecuda_evk *k) {
    if (!k) return HECUDA_OK;
    if (k->owner) pir_graphs_purge(const_cast<hecuda_context *>(k->owner), k);
    if (k->d_relin) cudaFree(k->d_relin);
    for (auto &kv : k->galois) cudaFree(kv.second);
    for (hecuda::u64 *p : k->retired) cudaFree(p);
    delete k;
    return HECUDA_OK;
}
int32_t hecuda_evk_device_buffer(hecuda_evk *k, void **device_ptr, uint64_t *bytes) {
    if (!k || !device_ptr || !bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *device_ptr = k->d_relin;
    *bytes = k->words * sizeof(u64);
    k->loaded = true;  // the caller fills it (e.g. ncclBroadcast from rank 0)
    ++k->version;
    return HECUDA_OK;
}

// ---------------------------------------------------------------- relinearize / mod switch

static int32_t check_relin(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l, uint64_t *out,
                           int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k || !k->loaded) return fail(HECUDA_ERR_MISSING_KEY, "missingRelinearizationKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (batch < 0 || (batch && (!ct3 || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    return HECUDA_OK;
}

int32_t hecuda_bfv_relinearize_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                                      uint64_t *out, int64_t batch, void *stream) {
    int32_t rc = check_relin(h, k, ct3, l, out, batch);
    if (rc) return rc;
    if (batch == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)3 * l * c.n, out_words = (size_t)2 * l * c.n;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, batch));
    cudaStream_t s = (cudaStream_t)stream;
    u64 *scratch = nullptr;
    CK(cudaMallocAsync(&scratch, relinearize_scratch_words(c, l) * (size_t)chunk * sizeof(u64), s));
    for (int64_t done = 0; done < batch; done += chunk) {
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        cudaError_t e = relinearize_chunk(c, scratch, k->d_relin, (const u64 *)ct3 + in_words * done, l,
                                          (u64 *)out + out_words * done, items, s);
        if (e != cudaSuccess) {
            cudaFreeAsync(scratch, s);
            return cuda_fail(e, "relinearize");
        }
    }
    CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}

int32_t hecuda_bfv_relinearize(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                               uint64_t *out, int64_t batch) {
    int32_t rc = check_relin(h, k, ct3, l, out, batch);
    if (rc) return rc;
    const Context &c = *h->ctx;
    std::vector<HostIo> in = {{(const u64 *)ct3, (size_t)3 * l * c.n}};
    return host_pipeline(h, batch, h->chunk, relinearize_scratch_words(c, l), in, (u64 *)out, (size_t)2 * l * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return relinearize_chunk(c, w.buf[0], k->d_relin, d_in[0], l, d_out, items, w.stream);
                         });
}

static int32_t check_ms(const hecuda_context *h, const uint64_t *ct, int32_t polys, int32_t l, uint64_t *out,
                        int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count");
    if (l < 2 || l > h->ctx->L)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (2 <= moduli_count <= L)");
    if (batch < 0 || (batch && (!ct || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    return HECUDA_OK;
}

int32_t hecuda_bfv_mod_switch_down_device(const hecuda_context *h, const uint64_t *ct, int32_t polys, int32_t l,
                                          uint64_t *out, int64_t batch, void *stream) {
    int32_t rc = check_ms(h, ct, polys, l, out, batch);
    if (rc) return rc;
    cudaError_t e = launch_mod_switch(*h->ctx, (const u64 *)ct, l, (u64 *)out, batch * polys, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "mod_switch");
    return HECUDA_OK;
}

int32_t hecuda_bfv_mod_switch_down(const hecuda_context *h, const uint64_t *ct, int32_t polys, int32_t l, uint64_t *out,
                                   int64_t batch) {
    int32_t rc = check_ms(h, ct, polys, l, out, batch);
    if (rc) return rc;
    const Context &c = *h->ctx;
    std::vector<HostIo> in = {{(const u64 *)ct, (size_t)polys * l * c.n}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / ((size_t)polys * l * c.n)));
    return host_pipeline(h, batch, chunk, 0, in, (u64 *)out, (size_t)polys * (l - 1) * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return launch_mod_switch(c, d_in[0], l, d_out, items * polys, w.stream);
                         });
}


// ---------------------------------------------------------------- relinearize -> modSwitchDown, fused
// Bfv.relinearize then Bfv.modSwitchDown on a batch in one pass (BASELINE config 3): the relinearized ciphertext stays
// in HBM, 2 x (l-1) rows per ciphertext come back.
int32_t hecuda_bfv_relinearize_mod_switch_down(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                                               uint64_t *out, int64_t batch) {
    int32_t rc = check_relin(h, k, ct3, l, out, batch);
    if (rc) return rc;
    if (l < 2) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (moduli_count >= 2)");
    const Context &c = *h->ctx;
    const size_t relin_words = (size_t)2 * l * c.n;
    std::vector<HostIo> in = {{(const u64 *)ct3, (size_t)3 * l * c.n}};
    return host_pipeline(h, batch, h->chunk, relinearize_scratch_words(c, l) + relin_words, in, (u64 *)out, (size_t)2 * (l - 1) * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             u64 *relin = w.buf[0] + relinearize_scratch_words(c, l) * (size_t)items;
                             cudaError_t e = relinearize_chunk(c, w.buf[0], k->d_relin, d_in[0], l, relin, items, w.stream);
                             if (e != cudaSuccess) return e;
                             return launch_mod_switch(c, relin, l, d_out, items * 2, w.stream);
                         });
}

// ---------------------------------------------------------------- multiply -> relinearize (-> modSwitchDown), fused
// The sequence every caller of ct x ct multiply runs (RlweBenchmark.swift:387-493; PirUtil.swift:447-480):
// Bfv.mulAssign, Bfv.relinearize, optionally Bfv.modSwitchDown, on a batch, in one pass: the three-polynomial product
// and the relinearized ciphertext stay in HBM and only 2 x L (or 2 x (L-1)) rows per ciphertext come back.
static size_t mul_relin_scratch_words(const Context &c) {
    // multiply scratch | 3-poly product | relinearize scratch | relinearized ciphertext (only with the modulus switch)
    return multiply_scratch_words(c) + (size_t)3 * c.L * c.n + relinearize_scratch_words(c, c.L) + (size_t)2 * c.L * c.n;
}
static cudaError_t mul_relin_chunk(const Context &c, u64 *scratch, const u64 *key, const u64 *lhs, const u64 *rhs, bool mod_switch,
                                   u64 *out, int64_t items, cudaStream_t s) {
    u64 *mul_scratch = scratch;
    u64 *prod = mul_scratch + multiply_scratch_words(c) * (size_t)items;
    u64 *ks_scratch = prod + (size_t)3 * c.L * c.n * items;
    u64 *relin = ks_scratch + relinearize_scratch_words(c, c.L) * (size_t)items;
    cudaError_t e;
    if ((e = multiply_chunk(c, mul_scratch, lhs, rhs, prod, items, s)) != cudaSuccess) return e;
    if ((e = relinearize_chunk(c, ks_scratch, key, prod, c.L, mod_switch ? relin : out, items, s)) != cudaSuccess) return e;
    if (mod_switch) return launch_mod_switch(c, relin, c.L, out, items * 2, s);
    return cudaSuccess;
}
static int32_t check_mul_relin(const hecuda_context *h, const hecuda_evk *k, const void *lhs, const void *rhs, const void *out,
                               int32_t mod_switch, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k || !k->loaded) return fail(HECUDA_ERR_MISSING_KEY, "missingRelinearizationKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (mod_switch && h->ctx->L < 2)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (L >= 2)");
    if (batch < 0 || (batch && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    return HECUDA_OK;
}
int32_t hecuda_bfv_multiply_relinearize_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *lhs,
                                               const uint64_t *rhs, int32_t mod_switch, uint64_t *out, int64_t batch,
                                               void *stream) {
    int32_t rc = check_mul_relin(h, k, lhs, rhs, out, mod_switch, batch);
    if (rc || batch == 0) return rc;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * (c.L - (mod_switch ? 1 : 0)) * c.n;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk / 2, batch));
    cudaStream_t s = (cudaStream_t)stream;
    u64 *scratch = nullptr;
    CK(cudaMallocAsync(&scratch, mul_relin_scratch_words(c) * (size_t)chunk * sizeof(u64), s));
    for (int64_t done = 0; done < batch; done += chunk) {
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        cudaError_t e = mul_relin_chunk(c, scratch, k->d_relin, (const u64 *)lhs + in_words * done, (const u64 *)rhs + in_words * done,
                                        mod_switch != 0, (u64 *)out + out_words * done, items, s);
        if (e != cudaSuccess) {
            cudaFreeAsync(scratch, s);
            return cuda_fail(e, "multiply_relinearize");
        }
    }
    CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}
int32_t hecuda_bfv_multiply_relinearize(const hecuda_context *h, const hecuda_evk *k, const uint64_t *lhs, const uint64_t *rhs,
                                        int32_t mod_switch, uint64_t *out, int64_t batch) {
    int32_t rc = check_mul_relin(h, k, lhs, rhs, out, mod_switch, batch);
    if (rc) return rc;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * (c.L - (mod_switch ? 1 : 0)) * c.n;
    std::vector<HostIo> in = {{(const u64 *)lhs, in_words}, {(const u64 *)rhs, in_words}};
    return host_pipeline(h, batch, std::max<int64_t>(1, h->chunk / 2), mul_relin_scratch_words(c), in, (u64 *)out, out_words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return mul_relin_chunk(c, w.buf[0], k->d_relin, d_in[0], d_in[1], mod_switch != 0, d_out, items,
                                                    w.stream);
                         });
}

// ---------------------------------------------------------------- Galois (SURVEY.md 8f rank 1)

static bool valid_galois_element(int64_t element, int64_t n) {  // isValidGaloisElement, Galois.swift:100-105
    return (element & 1) && element > 1 && element < 2 * n;
}

int32_t hecuda_evk_set_galois_key(hecuda_evk *k, uint32_t element, const uint64_t *key) {
    if (!k || !key) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_ctx(k->owner);
    if (rc) return rc;
    if (!valid_galois_element(element, k->owner->ctx->n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element");
    u64 *d = nullptr;
    CK(cudaMalloc(&d, k->words * sizeof(u64)));
    cudaError_t e = upload(d, key, k->words * sizeof(u64));
    if (e != cudaSuccess) {
        cudaFree(d);
        return cuda_fail(e, "cudaMemcpy(galois key)");
    }
    std::lock_guard<std::mutex> g(k->mu);
    auto it = k->galois.find(element);
    if (it != k->galois.end()) {
        // kernels already enqueued by other threads may still read the key being replaced (callers copy the device
        // pointer out under the mutex and launch afterwards): retire the buffer, free it with the handle
        k->retired.push_back(it->second);
        it->second = d;
    } else {
        k->galois[element] = d;
    }
    ++k->version;  // captured pipelines (pir.cu) bake the key pointers in: they are rebuilt on the next call
    return HECUDA_OK;
}

int32_t hecuda_evk_galois_device_buffer(hecuda_evk *k, uint32_t element, void **device_ptr, uint64_t *bytes) {
    if (!k || !device_ptr || !bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_ctx(k->owner);
    if (rc) return rc;
    if (!valid_galois_element(element, k->owner->ctx->n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element");
    std::lock_guard<std::mutex> g(k->mu);
    auto it = k->galois.find(element);
    if (it == k->galois.end()) {  // the caller fills it (e.g. ncclBroadcast from the rank that holds the key)
        u64 *d = nullptr;
        CK(cudaMalloc(&d, k->words * sizeof(u64)));
        it = k->galois.emplace(element, d).first;
    }
    *device_ptr = it->second;
    *bytes = k->words * sizeof(u64);
    return HECUDA_OK;
}

// EvaluationKey(deserialize:context:) (SerializedKeys.swift:141-157) with every key ciphertext .seeded: one DRBG chain
// pass over all the key's seeds, then one fused kernel that writes poly0 and poly1 of every ciphertext into the key's
// device buffers (drbg.cu).
int32_t hecuda_evk_create_serialized(const hecuda_context *h, const uint8_t *relin_poly0, const uint8_t *relin_seeds,
                                     const uint32_t *elements, int32_t element_count, const uint8_t *galois_poly0,
                                     const uint8_t *galois_seeds, hecuda_evk **out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    const Context &c = *h->ctx;
    if (!c.has_ks)
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: a single coefficient modulus leaves no key-switching modulus");
    if ((relin_poly0 == nullptr) != (relin_seeds == nullptr))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "relin_poly0 and relin_seeds must both be given or both be null");
    if (element_count < 0 || (element_count > 0 && (!elements || !galois_poly0 || !galois_seeds)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    std::vector<uint32_t> sorted(elements, elements + element_count);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t e : sorted)
        if (!valid_galois_element(e, c.n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element " + std::to_string(e));
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "repeated Galois element " + std::to_string(*std::adjacent_find(sorted.begin(), sorted.end())));
    uint64_t poly_bytes = 0;
    if ((rc = hecuda_poly_serialized_byte_count(h, HECUDA_BASE_KEYSWITCH, c.L + 1, 0, &poly_bytes))) return rc;
    const bool relin = relin_poly0 != nullptr;
    const int64_t count = (int64_t)(relin + element_count) * c.L;  // key ciphertexts
    hecuda_evk *k = nullptr;
    if ((rc = hecuda_evk_create_empty(h, &k))) return rc;
    // ciphertext i of key j lands at key_j + i x 2 x K x N: the relinearization key, then galois[elements[e]]
    std::vector<u64 *> dst;
    dst.reserve((size_t)count);
    const size_t ct_words = k->words / c.L;
    cudaError_t e = cudaSuccess;
    for (int32_t j = -1; j < element_count && e == cudaSuccess; ++j) {
        u64 *key = nullptr;
        if (j < 0) {
            if (!relin) continue;
            key = k->d_relin;
        } else if ((e = cudaMalloc(&key, k->words * sizeof(u64))) == cudaSuccess) {
            k->galois[elements[j]] = key;
        }
        for (int i = 0; key && i < c.L; ++i) dst.push_back(key + ct_words * i);
    }
    if (e == cudaSuccess && count > 0) {
        WsGuard g(h);
        if (!g.w) {
            hecuda_evk_destroy(k);
            return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
        }
        cudaStream_t s = g.w->stream;
        const size_t relin_cts = relin ? (size_t)c.L : 0, galois_cts = (size_t)element_count * c.L;
        unsigned char *d_poly0 = nullptr, *d_seeds = nullptr;
        u64 **d_dst = nullptr;
        e = cudaMallocAsync((void **)&d_poly0, poly_bytes * count, s);
        if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_seeds, (size_t)32 * count, s);
        if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_dst, sizeof(u64 *) * count, s);
        if (e == cudaSuccess && relin) e = cudaMemcpyAsync(d_poly0, relin_poly0, poly_bytes * relin_cts, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && relin) e = cudaMemcpyAsync(d_seeds, relin_seeds, 32 * relin_cts, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && galois_cts)
            e = cudaMemcpyAsync(d_poly0 + poly_bytes * relin_cts, galois_poly0, poly_bytes * galois_cts, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && galois_cts)
            e = cudaMemcpyAsync(d_seeds + 32 * relin_cts, galois_seeds, 32 * galois_cts, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_dst, dst.data(), sizeof(u64 *) * count, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = expand_seeded_keys_device(c, d_poly0, d_seeds, d_dst, count, s);
        for (void *p : {(void *)d_poly0, (void *)d_seeds, (void *)d_dst})
            if (p) cudaFreeAsync(p, s);
        // the keys are read on other non-blocking streams: return once the kernel has written them (see upload())
        const cudaError_t e2 = wait_stream(s);
        if (e == cudaSuccess) e = e2;
    }
    if (e != cudaSuccess) {
        hecuda_evk_destroy(k);
        return cuda_fail(e, "evk_create_serialized");
    }
    k->loaded = relin;
    *out = k;
    return HECUDA_OK;
}

static int32_t check_galois(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct, int32_t l, uint32_t element,
                            uint64_t *out, int64_t batch, const u64 **key) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (!valid_galois_element(element, h->ctx->n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element");
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (batch < 0 || (batch && (!ct || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    hecuda_evk *km = const_cast<hecuda_evk *>(k);
    std::lock_guard<std::mutex> g(km->mu);
    auto it = km->galois.find(element);
    if (it == km->galois.end()) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisElement: " + std::to_string(element));
    *key = it->second;
    return HECUDA_OK;
}

int32_t hecuda_bfv_apply_galois_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct, int32_t l,
                                       uint32_t element, uint64_t *out, int64_t batch, void *stream) {
    const u64 *key = nullptr;
    int32_t rc = check_galois(h, k, ct, l, element, out, batch, &key);
    if (rc) return rc;
    if (batch == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const size_t words = (size_t)2 * l * c.n;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, batch));
    cudaStream_t s = (cudaStream_t)stream;
    u64 *scratch = nullptr;
    CK(cudaMallocAsync(&scratch, galois_scratch_words(c, l) * (size_t)chunk * sizeof(u64), s));
    for (int64_t done = 0; done < batch; done += chunk) {
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        cudaError_t e = apply_galois_chunk(c, scratch, key, (const u64 *)ct + words * done, l, element,
                                           (u64 *)out + words * done, items, s);
        if (e != cudaSuccess) {
            cudaFreeAsync(scratch, s);
            return cuda_fail(e, "applyGalois");
        }
    }
    CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}

int32_t hecuda_bfv_apply_galois(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct, int32_t l,
                                uint32_t element, uint64_t *out, int64_t batch) {
    const u64 *key = nullptr;
    int32_t rc = check_galois(h, k, ct, l, element, out, batch, &key);
    if (rc) return rc;
    const Context &c = *h->ctx;
    std::vector<HostIo> in = {{(const u64 *)ct, (size_t)2 * l * c.n}};
    return host_pipeline(h, batch, h->chunk, galois_scratch_words(c, l), in, (u64 *)out, (size_t)2 * l * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return apply_galois_chunk(c, w.buf[0], key, d_in[0], l, element, d_out, items, w.stream);
                         });
}

int32_t hecuda_poly_apply_galois(const hecuda_context *h, int32_t base, int32_t eval_format, const uint64_t *in,
                                 uint64_t *out, int32_t rows, int64_t polys, uint32_t element) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (polys && (!in || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    if (!valid_galois_element(element, h->ctx->n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const Context &c = *h->ctx;
    const size_t words = (size_t)rows * c.n;
    std::vector<HostIo> hin = {{(const u64 *)in, words}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / words));
    return host_pipeline(h, polys, chunk, 0, hin, (u64 *)out, words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return eval_format ? launch_galois_eval(c, rows, element, d_in[0], d_out, items, w.stream)
                                                : launch_galois_coeff(c, map, element, d_in[0], (int64_t)words, d_out,
                                                                      (int64_t)words, items, w.stream);
                         });
}

// ---------------------------------------------------------------- lazy ct x pt inner product (SURVEY.md 8f rank 2)

static int32_t check_ip(const hecuda_context *h, const uint64_t *cts, int32_t polys, int32_t l, int64_t terms,
                        const uint64_t *pts, uint64_t *out, int64_t out_count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 1 || polys > 3) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count must be 1..3");
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (terms < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "Empty ciphertexts");  // precondition, Bfv.swift:481-483
    if (out_count < 0 || (out_count && (!cts || !pts || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    if (h->ctx->n < 2) return fail(HECUDA_ERR_UNSUPPORTED, "degree too small");
    return HECUDA_OK;
}

int32_t hecuda_bfv_inner_product_plaintexts_device(const hecuda_context *h, const uint64_t *cts, int32_t polys,
                                                   int32_t l, int64_t terms, const uint64_t *pts,
                                                   const uint8_t *present, uint64_t *out, int64_t out_count,
                                                   void *stream) {
    int32_t rc = check_ip(h, cts, polys, l, terms, pts, out, out_count);
    if (rc) return rc;
    cudaError_t e = launch_inner_product_plain(*h->ctx, (const u64 *)cts, polys, l, terms, (const u64 *)pts, present,
                                               (u64 *)out, out_count, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "inner_product");
    return HECUDA_OK;
}

int32_t hecuda_bfv_inner_product_plaintexts(const hecuda_context *h, const uint64_t *cts, int32_t polys, int32_t l,
                                            int64_t terms, const uint64_t *pts, const uint8_t *present, uint64_t *out,
                                            int64_t out_count) {
    int32_t rc = check_ip(h, cts, polys, l, terms, pts, out, out_count);
    if (rc) return rc;
    if (out_count == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    // the query ciphertexts (and the presence flags) are shared by every output row: upload once
    const size_t ct_words = (size_t)terms * polys * l * c.n;
    u64 *d_cts = nullptr;
    unsigned char *d_present = nullptr;
    CK(cudaMalloc(&d_cts, ct_words * sizeof(u64)));
    cudaError_t e = upload(d_cts, cts, ct_words * sizeof(u64));
    if (e == cudaSuccess && present) {
        e = cudaMalloc(&d_present, (size_t)out_count * terms);
        if (e == cudaSuccess) e = upload(d_present, present, (size_t)out_count * terms);
    }
    if (e != cudaSuccess) {
        cudaFree(d_cts);
        cudaFree(d_present);
        return cuda_fail(e, "inner_product upload");
    }
    const size_t pt_words = (size_t)terms * l * c.n;
    std::vector<HostIo> in = {{(const u64 *)pts, pt_words}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)32 * 1024 * 1024 / pt_words));
    int64_t done_items = 0;  // host_pipeline calls the body in order, one chunk at a time
    rc = host_pipeline(h, out_count, chunk, 0, in, (u64 *)out, (size_t)polys * l * c.n,
                       [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                           const unsigned char *pr = d_present ? d_present + done_items * terms : nullptr;
                           done_items += items;
                           return launch_inner_product_plain(c, d_cts, polys, l, terms, d_in[0], pr, d_out, items, w.stream);
                       });
    cudaDeviceSynchronize();
    cudaFree(d_cts);
    cudaFree(d_present);
    return rc;
}

int32_t hecuda_plaintext_to_eval_device(const hecuda_context *h, const uint64_t *plain, int32_t l, uint64_t *out,
                                        int64_t count, void *stream) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count out of range");
    if (count < 0 || (count && (!plain || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    cudaError_t e = launch_plaintext_to_eval(*h->ctx, (const u64 *)plain, l, (u64 *)out, count, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "plaintext_to_eval");
    return HECUDA_OK;
}

int32_t hecuda_plaintext_to_eval(const hecuda_context *h, const uint64_t *plain, int32_t l, uint64_t *out,
                                 int64_t count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count out of range");
    if (count < 0 || (count && (!plain || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    const Context &c = *h->ctx;
    std::vector<HostIo> in = {{(const u64 *)plain, (size_t)c.n}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / ((size_t)l * c.n)));
    return host_pipeline(h, count, chunk, 0, in, (u64 *)out, (size_t)l * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return launch_plaintext_to_eval(c, d_in[0], l, d_out, items, w.stream);
                         });
}

// ---------------------------------------------------------------- plaintext side: SIMD encode / decode, ct +- pt

int32_t hecuda_context_supports_simd(const hecuda_context *h, int32_t *supported) {
    if (!h || !h->ctx || !supported) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *supported = h->ctx->simd ? 1 : 0;
    return HECUDA_OK;
}

}  // extern "C"

namespace {

int32_t need_simd(const hecuda_context *h) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!h->ctx->simd)
        return fail(HECUDA_ERR_UNSUPPORTED, "simdEncodingNotSupported: the plaintext modulus is not a prime = 1 mod 2N");
    return HECUDA_OK;
}

// encodingDataOutOfBounds (Encoding.swift:147-156): host buffers of uint64 (or uint32 inside a hecuda_u32_ call)
bool host_values_below(const void *p, size_t count, u64 t) {
    if (tl_io32) {
        const uint32_t *v = static_cast<const uint32_t *>(p);
        return std::all_of(v, v + count, [t](uint32_t x) { return x < t; });
    }
    const uint64_t *v = static_cast<const uint64_t *>(p);
    return std::all_of(v, v + count, [t](uint64_t x) { return x < t; });
}

int32_t check_encode(const hecuda_context *h, const void *values, int32_t value_count, int32_t l, const void *out,
                     int64_t count) {
    int32_t rc = need_simd(h);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (value_count < 0 || value_count > c.n)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "encodingDataCountExceedsLimit: value_count must be in [0, N]");
    if (l < 0 || l > c.L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count must be in [0, L]");
    if (count < 0 || (count && (!out || (value_count && !values)))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    return HECUDA_OK;
}

int32_t check_decode(const hecuda_context *h, const void *plain, int32_t l, const void *values, int64_t count) {
    int32_t rc = need_simd(h);
    if (rc) return rc;
    if (l < 0 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count must be in [0, L]");
    if (count < 0 || (count && (!plain || !values))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    return HECUDA_OK;
}

int32_t check_translate(const hecuda_context *h, const void *ct, int32_t polys, int32_t l, const void *pt, int64_t pt_count,
                        int32_t op, const void *out, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 2 || polys > 3) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count must be 2 or 3");
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count must be in [1, L]");
    if (op < HECUDA_PLAINTEXT_ADD || op > HECUDA_PLAINTEXT_SUB_FROM) return fail(HECUDA_ERR_INVALID_ARGUMENT, "unknown op");
    if (batch < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: negative batch");
    if (pt_count != 1 && pt_count != batch)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "incompatibleCiphertextAndPlaintext: plaintext_count must be 1 or batch");
    if (batch && (!ct || !pt || !out)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    return HECUDA_OK;
}

// items per device-side chunk of the encode / decode pipelines: scratch of at most 2^25 words
int64_t simd_chunk(const Context &c) { return std::max<int64_t>(1, ((int64_t)1 << 25) / c.n); }

}  // namespace

extern "C" {

int32_t hecuda_bfv_encode_simd_device(const hecuda_context *h, const uint64_t *values, int32_t value_count,
                                      int32_t moduli_count, uint64_t *out, int64_t count, void *stream) {
    int32_t rc = check_encode(h, values, value_count, moduli_count, out, count);
    if (rc || count == 0) return rc;
    const Context &c = *h->ctx;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t chunk = std::min<int64_t>(simd_chunk(c), count);
    const size_t scratch_words = simd_scratch_words(c, true, moduli_count) * (size_t)chunk;
    u64 *scratch = nullptr;
    if (scratch_words) CK(cudaMallocAsync(&scratch, scratch_words * sizeof(u64), s));
    const int64_t out_words = (int64_t)(moduli_count ? moduli_count : 1) * c.n;
    cudaError_t e = cudaSuccess;
    for (int64_t done = 0; e == cudaSuccess && done < count; done += chunk)
        e = launch_encode_simd(c, (const u64 *)values + done * value_count, value_count, moduli_count,
                               (u64 *)out + done * out_words, scratch, std::min<int64_t>(chunk, count - done), s);
    if (scratch) cudaFreeAsync(scratch, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "encodeSimd");
}

int32_t hecuda_bfv_encode_simd(const hecuda_context *h, const uint64_t *values, int32_t value_count, int32_t moduli_count,
                               uint64_t *out, int64_t count) {
    int32_t rc = check_encode(h, values, value_count, moduli_count, out, count);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!host_values_below(values, (size_t)count * value_count, c.t))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "encodingDataOutOfBounds: values must be below the plaintext modulus");
    const int l = moduli_count;
    std::vector<HostIo> in;
    if (value_count) in.push_back({(const u64 *)values, (size_t)value_count});
    const size_t out_words = (size_t)(l ? l : 1) * c.n;
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / out_words));
    return host_pipeline(h, count, chunk, simd_scratch_words(c, true, l), in, (u64 *)out, out_words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return launch_encode_simd(c, d_in.empty() ? nullptr : d_in[0], value_count, l, d_out, w.buf[0],
                                                       items, w.stream);
                         });
}

int32_t hecuda_bfv_decode_simd_device(const hecuda_context *h, const uint64_t *plaintexts, int32_t moduli_count,
                                      uint64_t *values, int64_t count, void *stream) {
    int32_t rc = check_decode(h, plaintexts, moduli_count, values, count);
    if (rc || count == 0) return rc;
    const Context &c = *h->ctx;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t chunk = std::min<int64_t>(simd_chunk(c), count);
    u64 *scratch = nullptr;
    CK(cudaMallocAsync(&scratch, simd_scratch_words(c, false, moduli_count) * (size_t)chunk * sizeof(u64), s));
    const int64_t in_words = (int64_t)(moduli_count ? moduli_count : 1) * c.n;
    cudaError_t e = cudaSuccess;
    for (int64_t done = 0; e == cudaSuccess && done < count; done += chunk)
        e = launch_decode_simd(c, (const u64 *)plaintexts + done * in_words, moduli_count, (u64 *)values + done * c.n, scratch,
                               std::min<int64_t>(chunk, count - done), s);
    cudaFreeAsync(scratch, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "decodeSimd");
}

int32_t hecuda_bfv_decode_simd(const hecuda_context *h, const uint64_t *plaintexts, int32_t moduli_count, uint64_t *values,
                               int64_t count) {
    int32_t rc = check_decode(h, plaintexts, moduli_count, values, count);
    if (rc) return rc;
    const Context &c = *h->ctx;
    const int l = moduli_count;
    const size_t in_words = (size_t)(l ? l : 1) * c.n;
    std::vector<HostIo> in = {{(const u64 *)plaintexts, in_words}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / in_words));
    return host_pipeline(h, count, chunk, simd_scratch_words(c, false, l), in, (u64 *)values, (size_t)c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return launch_decode_simd(c, d_in[0], l, d_out, w.buf[0], items, w.stream);
                         });
}

int32_t hecuda_bfv_plaintext_translate_device(const hecuda_context *h, const uint64_t *ct, int32_t poly_count,
                                              int32_t moduli_count, const uint64_t *plaintexts, int64_t plaintext_count,
                                              int32_t op, uint64_t *out, int64_t batch, void *stream) {
    int32_t rc = check_translate(h, ct, poly_count, moduli_count, plaintexts, plaintext_count, op, out, batch);
    if (rc) return rc;
    cudaError_t e = launch_plaintext_translate(*h->ctx, (const u64 *)ct, poly_count, moduli_count, (const u64 *)plaintexts,
                                               plaintext_count == 1, op, (u64 *)out, batch, (cudaStream_t)stream);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "plaintextTranslate");
}

int32_t hecuda_bfv_plaintext_translate(const hecuda_context *h, const uint64_t *ct, int32_t poly_count, int32_t moduli_count,
                                       const uint64_t *plaintexts, int64_t plaintext_count, int32_t op, uint64_t *out,
                                       int64_t batch) {
    int32_t rc = check_translate(h, ct, poly_count, moduli_count, plaintexts, plaintext_count, op, out, batch);
    if (rc || batch == 0) return rc;
    const Context &c = *h->ctx;
    if (!host_values_below(plaintexts, (size_t)plaintext_count * c.n, c.t))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "encodingDataOutOfBounds: plaintext coefficients must be below t");
    const bool broadcast = plaintext_count == 1;
    const int l = moduli_count;
    const size_t ct_words = (size_t)poly_count * l * c.n;
    std::vector<HostIo> in = {{(const u64 *)ct, ct_words}};
    u64 *d_pt = nullptr;  // the shared plaintext, uploaded once
    if (broadcast) {
        std::vector<u64> pt(c.n);
        if (tl_io32) std::copy((const uint32_t *)plaintexts, (const uint32_t *)plaintexts + c.n, pt.begin());
        else std::copy(plaintexts, plaintexts + c.n, pt.begin());
        CK(cudaMalloc(&d_pt, sizeof(u64) * (size_t)c.n));
        cudaError_t e = upload(d_pt, pt.data(), sizeof(u64) * (size_t)c.n);
        if (e != cudaSuccess) {
            cudaFree(d_pt);
            return cuda_fail(e, "plaintext upload");
        }
    } else {
        in.push_back({(const u64 *)plaintexts, (size_t)c.n});
    }
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / ct_words));
    rc = host_pipeline(h, batch, chunk, 0, in, (u64 *)out, ct_words,
                       [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                           return launch_plaintext_translate(c, d_in[0], poly_count, l, broadcast ? d_pt : d_in[1], broadcast,
                                                             op, d_out, items, w.stream);
                       });
    if (d_pt) cudaFree(d_pt);
    return rc;
}

// ---------------------------------------------------------------- ct x ct inner product (SURVEY.md 8f rank 2)

static int32_t check_ipc(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out, int64_t pairs,
                         int64_t groups) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (pairs < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "Empty ciphertexts");
    if (groups < 0 || (groups && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    if (h->ctx->n < 2) return fail(HECUDA_ERR_UNSUPPORTED, "degree too small");
    return HECUDA_OK;
}

int32_t hecuda_bfv_inner_product_device(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                        int64_t pairs, int64_t groups, void *stream) {
    int32_t rc = check_ipc(h, lhs, rhs, out, pairs, groups);
    if (rc) return rc;
    if (groups == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)pairs * 2 * c.L * c.n, out_words = (size_t)3 * c.L * c.n;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(1, h->chunk / pairs), groups));
    cudaStream_t s = (cudaStream_t)stream;
    u64 *scratch = nullptr;
    CK(cudaMallocAsync(&scratch, inner_product_scratch_words(c, pairs) * (size_t)chunk * sizeof(u64), s));
    for (int64_t done = 0; done < groups; done += chunk) {
        const int64_t g = std::min<int64_t>(chunk, groups - done);
        cudaError_t e = inner_product_chunk(c, scratch, (const u64 *)lhs + in_words * done, (const u64 *)rhs + in_words * done,
                                            pairs, (u64 *)out + out_words * done, g, s);
        if (e != cudaSuccess) {
            cudaFreeAsync(scratch, s);
            return cuda_fail(e, "innerProduct");
        }
    }
    CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}

int32_t hecuda_bfv_inner_product(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                 int64_t pairs, int64_t groups) {
    int32_t rc = check_ipc(h, lhs, rhs, out, pairs, groups);
    if (rc) return rc;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)pairs * 2 * c.L * c.n;
    std::vector<HostIo> in = {{(const u64 *)lhs, in_words}, {(const u64 *)rhs, in_words}};
    const int64_t chunk = std::max<int64_t>(1, h->chunk / pairs);
    return host_pipeline(h, groups, chunk, inner_product_scratch_words(c, pairs), in, (u64 *)out, (size_t)3 * c.L * c.n,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t g) {
                             return inner_product_chunk(c, w.buf[0], d_in[0], d_in[1], pairs, d_out, g, w.stream);
                         });
}

int32_t hecuda_poly_multiply_power_of_x(const hecuda_context *h, int32_t base, const uint64_t *in, uint64_t *out,
                                        int32_t rows, int64_t polys, int64_t power) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (polys && (!in || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const Context &c = *h->ctx;
    const size_t words = (size_t)rows * c.n;
    std::vector<HostIo> hin = {{(const u64 *)in, words}};
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)4 * 1024 * 1024 / words));
    return host_pipeline(h, polys, chunk, 0, hin, (u64 *)out, words,
                         [&](Workspace &w, const std::vector<const u64 *> &d_in, u64 *d_out, int64_t items) {
                             return launch_multiply_power_of_x(c, map, power, d_in[0], d_out, items, w.stream);
                         });
}

uint64_t hecuda_kernel_launch_count(void) { return g_kernel_launches.load(); }


// ---------------------------------------------------------------- Bfv<UInt32>: uint32 buffers at the boundary
// (the reference's second scalar type, HeScheme.swift / Scalar.swift:498-511).  Same layouts as the uint64 entry points;
// the context must have been made by hecuda_context_create_u32 (its m~, gamma and Bsk).
static int32_t need_word32(const hecuda_context *h) {
    if (!h || !h->ctx) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: null context");
    if (h->ctx->word_bits != 32) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: not a Bfv<UInt32> context (hecuda_context_create_u32)");
    return HECUDA_OK;
}
int32_t hecuda_u32_ntt_forward(const hecuda_context *h, int32_t base, uint32_t *data, int32_t rows, int64_t polys) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_ntt_forward(h, base, reinterpret_cast<uint64_t *>(data), rows, polys);
}
int32_t hecuda_u32_ntt_inverse(const hecuda_context *h, int32_t base, uint32_t *data, int32_t rows, int64_t polys) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_ntt_inverse(h, base, reinterpret_cast<uint64_t *>(data), rows, polys);
}
int32_t hecuda_u32_bfv_multiply(const hecuda_context *h, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_multiply(h, reinterpret_cast<const uint64_t *>(lhs), reinterpret_cast<const uint64_t *>(rhs),
                               reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_evk_create(const hecuda_context *h, const uint32_t *relin_key, hecuda_evk **out) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    if (!relin_key) return fail(HECUDA_ERR_MISSING_KEY, "missingRelinearizationKey");
    const Context &c = *h->ctx;
    const size_t words = (size_t)c.L * 2 * (c.L + 1) * c.n;
    std::vector<uint64_t> wide(relin_key, relin_key + words);  // setup-time: widened on the host
    return hecuda_evk_create(h, wide.data(), out);
}
int32_t hecuda_u32_bfv_relinearize(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *ct3, int32_t l, uint32_t *out,
                                   int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_relinearize(h, evk, reinterpret_cast<const uint64_t *>(ct3), l, reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_bfv_mod_switch_down(const hecuda_context *h, const uint32_t *ct, int32_t polys, int32_t l, uint32_t *out,
                                       int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_mod_switch_down(h, reinterpret_cast<const uint64_t *>(ct), polys, l, reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_bfv_multiply_relinearize(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *lhs, const uint32_t *rhs,
                                            int32_t mod_switch, uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_multiply_relinearize(h, evk, reinterpret_cast<const uint64_t *>(lhs), reinterpret_cast<const uint64_t *>(rhs),
                                           mod_switch, reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_bfv_relinearize_mod_switch_down(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *ct3, int32_t l,
                                                   uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_relinearize_mod_switch_down(h, evk, reinterpret_cast<const uint64_t *>(ct3), l,
                                                  reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_evk_set_galois_key(hecuda_evk *evk, uint32_t element, const uint32_t *key) {
    if (!evk || !key) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = need_word32(evk->owner);
    if (rc) return rc;
    std::vector<uint64_t> wide(key, key + evk->words);  // setup-time: widened on the host
    return hecuda_evk_set_galois_key(evk, element, wide.data());
}
int32_t hecuda_u32_bfv_apply_galois(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *ct, int32_t l, uint32_t element,
                                    uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_apply_galois(h, evk, reinterpret_cast<const uint64_t *>(ct), l, element, reinterpret_cast<uint64_t *>(out), batch);
}
int32_t hecuda_u32_bfv_inner_product(const hecuda_context *h, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out, int64_t pairs,
                                     int64_t groups) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_inner_product(h, reinterpret_cast<const uint64_t *>(lhs), reinterpret_cast<const uint64_t *>(rhs),
                                    reinterpret_cast<uint64_t *>(out), pairs, groups);
}
int32_t hecuda_u32_rnstool_lift_q_to_qbsk(const hecuda_context *h, const uint32_t *polys, uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_rnstool_lift_q_to_qbsk(h, reinterpret_cast<const uint64_t *>(polys), reinterpret_cast<uint64_t *>(out), count);
}
int32_t hecuda_u32_rnstool_floor_qbsk_to_q(const hecuda_context *h, const uint32_t *polys, uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_rnstool_floor_qbsk_to_q(h, reinterpret_cast<const uint64_t *>(polys), reinterpret_cast<uint64_t *>(out), count);
}
int32_t hecuda_u32_bfv_encode_simd(const hecuda_context *h, const uint32_t *values, int32_t value_count, int32_t moduli_count,
                                   uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_encode_simd(h, reinterpret_cast<const uint64_t *>(values), value_count, moduli_count,
                                  reinterpret_cast<uint64_t *>(out), count);
}
int32_t hecuda_u32_bfv_decode_simd(const hecuda_context *h, const uint32_t *plaintexts, int32_t moduli_count, uint32_t *values,
                                   int64_t count) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_decode_simd(h, reinterpret_cast<const uint64_t *>(plaintexts), moduli_count,
                                  reinterpret_cast<uint64_t *>(values), count);
}
int32_t hecuda_u32_bfv_plaintext_translate(const hecuda_context *h, const uint32_t *ct, int32_t poly_count, int32_t moduli_count,
                                           const uint32_t *plaintexts, int64_t plaintext_count, int32_t op, uint32_t *out,
                                           int64_t batch) {
    int32_t rc = need_word32(h);
    if (rc) return rc;
    Io32Scope scope;
    return hecuda_bfv_plaintext_translate(h, reinterpret_cast<const uint64_t *>(ct), poly_count, moduli_count,
                                          reinterpret_cast<const uint64_t *>(plaintexts), plaintext_count, op,
                                          reinterpret_cast<uint64_t *>(out), batch);
}

}  // extern "C"
