// capi.cu -- the C ABI declared in include/hecuda.h.  No torch types, no exceptions across the boundary.
//
// Each batched operation is described once (a Batched: per-item buffer sizes, chunk sizes and a body that runs a run of
// items on the device) and run three ways.  Host-pointer entry points run it through a pipeline of three workspaces on
// three streams, so that the H2D copy of stage k+1, the kernels of stage k and the D2H copy of stage k-1 overlap when
// the caller's buffers are pinned; the hecuda_u32_ entry points run the same pipeline on uint32 host buffers.
// Device-pointer entry points enqueue on the caller's stream and do not synchronize.
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
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "capi_internal.hpp"
#include "pir_proto.hpp"

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
// then ONE dropExtendedBase -- instead of `pairs` full multiplies.  The sum grows with `pairs`; past aux_max_pairs it
// would wrap in the auxiliary base (context.cu), so it runs over the reference's Bsk, as the reference does.  The floor's
// folded Q-row scaling (kScaleTMontFloor) lives in the Q slots' inverse twiddles and is the same for either base.
cudaError_t inner_product_chunk(const Context &c, u64 *scratch, const u64 *lhs, const u64 *rhs, int64_t pairs,
                                       u64 *out, int64_t groups, cudaStream_t s) {
    const int R = 2 * c.L + 1;
    const size_t poly_words = (size_t)R * c.n;
    const int64_t items = groups * pairs;
    u64 *ext = scratch, *ten = scratch + 4 * poly_words * items;
    const bool bsk = pairs > c.aux_max_pairs;
    const NttRowMap map = bsk ? c.map_qbsk() : c.map_qaux();
    cudaError_t e;
    const bool scaled = floor_takes_scaled_q(c);
    if ((e = launch_lift(c, lhs, rhs, 2, ext, items, s, bsk)) != cudaSuccess) return e;
    if ((e = launch_ntt_forward(c, map, ext, ext, items * 4 * R, s)) != cudaSuccess) return e;
    if ((e = launch_tensor_sum(c, ext, ten, pairs, groups, s, bsk)) != cudaSuccess) return e;
    if ((e = launch_ntt_inverse(c, map, ten, ten, groups * 3 * R, scaled ? kScaleTMontFloor : kScaleTMont, s)) != cudaSuccess)
        return e;
    return launch_floor(c, ten, out, groups * 3, s, bsk, scaled);
}
size_t inner_product_scratch_words(const Context &c, int64_t pairs) {
    return (size_t)(4 * pairs + 3) * (2 * c.L + 1) * c.n;
}

}  // namespace api
}  // namespace hecuda

namespace {

// Host buffers of uint64 words, or of uint32 words in the hecuda_u32_ entry points (Bfv<UInt32> contexts): the host
// pipeline widens those after the H2D copy and narrows the output before the D2H copy.
enum class Words { u64, u32 };

constexpr int kPipelineDepth = 3;              // host pipeline stages in flight, each on its own stream
constexpr int64_t kMinStages = 16;             // a batch of 64 or more runs in at least this many stages of >= 16 items
constexpr size_t kStageWords = 4 * 1024 * 1024;  // per-stage budget of the operations not sized by h->chunk
constexpr int64_t kWholeBatch = INT64_MAX;     // items per device launch of the operations that launch once

// items per stage when the largest per-item buffer is `words`
int64_t stage_items(size_t budget, size_t words) { return std::max<int64_t>(1, (int64_t)(budget / words)); }

// One run of items [first, first + items) of a Batched: in[i] and out point at item `first`, scratch holds
// items x scratch_words.
struct Chunk {
    u64 *scratch;
    int64_t first, items;
    const u64 *const *in;
    u64 *out;
    cudaStream_t stream;
};

// One batched operation.  Items lie back to back in every input and in the output; operands shared by every item
// are uploaded once by the caller and captured by the body.
struct Batched {
    const char *name;  // in the device entry points' errors
    struct Io {
        const void *p;  // host (uint64 or uint32 words) or device buffer
        size_t words;   // per item
    };
    std::vector<Io> in;
    void *out;
    size_t out_words, scratch_words;  // per item
    int64_t per_launch;               // items per device launch
    int64_t stage_hint;               // items per host pipeline stage, before host_pipeline's clamp
    std::function<cudaError_t(const Chunk &)> body;
};

// On the caller's device buffers and stream: per_launch items per body call, no host synchronisation, stream-ordered
// scratch (graph-capturable), nothing launched for an empty batch.
int32_t run_device(const Batched &op, int64_t batch, cudaStream_t s) {
    if (batch == 0) return HECUDA_OK;
    const int64_t chunk = std::min(op.per_launch, batch);
    u64 *scratch = nullptr;
    if (op.scratch_words) CK(cudaMallocAsync(&scratch, op.scratch_words * (size_t)chunk * sizeof(u64), s));
    std::vector<const u64 *> in(op.in.size());
    cudaError_t e = cudaSuccess;
    for (int64_t done = 0; e == cudaSuccess && done < batch; done += chunk) {
        for (size_t i = 0; i < in.size(); ++i) in[i] = static_cast<const u64 *>(op.in[i].p) + op.in[i].words * (size_t)done;
        e = op.body({scratch, done, std::min(chunk, batch - done), in.data(),
                     static_cast<u64 *>(op.out) + op.out_words * (size_t)done, s});
    }
    if (e != cudaSuccess) {
        if (scratch) cudaFreeAsync(scratch, s);
        return cuda_fail(e, op.name);
    }
    if (scratch) CK(cudaFreeAsync(scratch, s));
    return HECUDA_OK;
}

// On host buffers: for each stage, copy the inputs in, run the body, copy the output out.
int32_t host_pipeline(const hecuda_context *h, const Batched &op, int64_t batch, Words words) {
    if (batch == 0) return HECUDA_OK;
    std::vector<std::unique_ptr<WsGuard>> guards;
    std::vector<Workspace *> ws;
    for (int i = 0; i < kPipelineDepth; ++i) {
        guards.emplace_back(new WsGuard(h));
        if (!guards.back()->w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
        ws.push_back(guards.back()->w);
    }
    int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(op.stage_hint, batch));
    if (batch >= 64) chunk = std::min<int64_t>(chunk, std::max<int64_t>(16, (batch + kMinStages - 1) / kMinStages));
    // On any early return, earlier stages may still have copies into / out of the caller's buffers in flight on the
    // other streams: wait for all of them so the caller may free or reuse its buffers as soon as it sees the error.
    struct DrainOnExit {
        std::vector<Workspace *> &ws;
        ~DrainOnExit() {
            for (Workspace *w : ws) wait_stream(w->stream);
        }
    } drain{ws};
    const bool io32 = words == Words::u32;
    int k = 0;
    for (int64_t done = 0; done < batch; done += chunk, ++k) {
        Workspace &w = *ws[k % kPipelineDepth];
        const int64_t items = std::min<int64_t>(chunk, batch - done);
        // Work on one workspace is ordered by its stream; buffers only ever grow (first kPipelineDepth stages).
        size_t in_words = 0;
        for (const Batched::Io &io : op.in) in_words += io.words * (size_t)items;
        const size_t out_words = op.out_words * (size_t)items;
        CK(w.scratch.reserve(op.scratch_words * (size_t)items));
        CK(w.in.reserve(in_words));
        CK(w.out.reserve(out_words));
        if (io32) {  // each input's uint32 image starts on a 16-byte boundary
            CK(w.in32.reserve(in_words / 2 + op.in.size() * 2 + 2));
            CK(w.out32.reserve(out_words / 2 + 2));
        }
        std::vector<const u64 *> d_in;
        size_t off = 0, off32 = 0;
        for (const Batched::Io &io : op.in) {
            const size_t n = io.words * (size_t)items, first = io.words * (size_t)done;
            if (io32) {
                u32 *raw = reinterpret_cast<u32 *>(w.in32.p) + off32;
                CK(cudaMemcpyAsync(raw, static_cast<const u32 *>(io.p) + first, n * sizeof(u32), cudaMemcpyHostToDevice,
                                   w.stream));
                CK(launch_widen(raw, w.in.p + off, (int64_t)n, w.stream));
                off32 += (n + 3) & ~(size_t)3;
            } else {
                CK(cudaMemcpyAsync(w.in.p + off, static_cast<const u64 *>(io.p) + first, n * sizeof(u64),
                                   cudaMemcpyHostToDevice, w.stream));
            }
            d_in.push_back(w.in.p + off);
            off += n;
        }
        cudaError_t e = op.body({w.scratch.p, done, items, d_in.data(), w.out.p, w.stream});
        if (e != cudaSuccess) return cuda_fail(e, "kernel launch");
        const size_t first = op.out_words * (size_t)done;
        if (io32) {
            u32 *out32 = reinterpret_cast<u32 *>(w.out32.p);
            CK(launch_narrow(w.out.p, out32, (int64_t)out_words, w.stream));
            CK(cudaMemcpyAsync(static_cast<u32 *>(op.out) + first, out32, out_words * sizeof(u32), cudaMemcpyDeviceToHost,
                               w.stream));
        } else {
            CK(cudaMemcpyAsync(static_cast<u64 *>(op.out) + first, w.out.p, out_words * sizeof(u64), cudaMemcpyDeviceToHost,
                               w.stream));
        }
    }
    for (Workspace *w : ws) CK(wait_stream(w->stream));
    return HECUDA_OK;
}

// Where a batched entry point runs its operation: on device buffers on the caller's stream, or through the host
// pipeline on host buffers of `words`.
struct Target {
    bool device;
    cudaStream_t stream;
    Words words;
};
constexpr Target kHost64{false, nullptr, Words::u64}, kHost32{false, nullptr, Words::u32};
Target on_stream(void *stream) { return {true, (cudaStream_t)stream, Words::u64}; }

int32_t run(const hecuda_context *h, const Batched &op, int64_t batch, Target t) {
    return t.device ? run_device(op, batch, t.stream) : host_pipeline(h, op, batch, t.words);
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

// forward or inverse NTT, in place, of items of `rows` rows
static Batched ntt_op(const Context &c, const NttRowMap &map, void *data, int64_t rows, bool inverse) {
    const size_t words = (size_t)rows * c.n;
    return {"ntt launch", {{data, words}}, data, words, 0, kWholeBatch, stage_items(kStageWords, words),
            [&c, map, rows, inverse](const Chunk &x) {
                return inverse ? launch_ntt_inverse(c, map, x.in[0], x.out, x.items * rows, kScalePlain, x.stream)
                               : launch_ntt_forward(c, map, x.in[0], x.out, x.items * rows, x.stream);
            }};
}
static int32_t ntt(const hecuda_context *h, int32_t base, void *data, int32_t rows, int64_t polys, bool inverse, Target t) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (!data && polys)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    return run(h, ntt_op(*h->ctx, map, data, rows, inverse), polys, t);
}
int32_t hecuda_ntt_forward_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys,
                                  void *stream) {
    return ntt(h, base, data, rows, polys, false, on_stream(stream));
}
int32_t hecuda_ntt_inverse_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys,
                                  void *stream) {
    return ntt(h, base, data, rows, polys, true, on_stream(stream));
}
int32_t hecuda_ntt_forward(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys) {
    return ntt(h, base, data, rows, polys, false, kHost64);
}
int32_t hecuda_ntt_inverse(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys) {
    return ntt(h, base, data, rows, polys, true, kHost64);
}
// Stage-level BEHZ entry points over the reference's [Q, Bsk] (RnsTool.swift:324-331, 453-456), Coeff format.
static int32_t lift_or_floor(const hecuda_context *h, const void *polys, void *out, int64_t count, bool lift, Words words) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (count < 0 || ((!polys || !out) && count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid buffers / poly_count");
    const Context &c = *h->ctx;
    const size_t q_words = (size_t)c.L * c.n, qbsk_words = (size_t)(2 * c.L + 1) * c.n;
    return host_pipeline(h,
                         {lift ? "lift" : "floor", {{polys, lift ? q_words : qbsk_words}}, out, lift ? qbsk_words : q_words, 0,
                          kWholeBatch, stage_items(kStageWords, qbsk_words),
                          [&](const Chunk &x) {
                              return lift ? launch_lift(c, x.in[0], nullptr, 1, x.out, x.items, x.stream, /*reference_base=*/true)
                                          : launch_floor(c, x.in[0], x.out, x.items, x.stream, /*reference_base=*/true);
                          }},
                         count, words);
}
int32_t hecuda_rnstool_lift_q_to_qbsk(const hecuda_context *h, const uint64_t *polys, uint64_t *out, int64_t count) {
    return lift_or_floor(h, polys, out, count, true, Words::u64);
}
int32_t hecuda_rnstool_floor_qbsk_to_q(const hecuda_context *h, const uint64_t *polys, uint64_t *out, int64_t count) {
    return lift_or_floor(h, polys, out, count, false, Words::u64);
}

static int32_t ntt_rows(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows, bool inverse) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (rows < 0 || (!data && rows)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / row_count");
    const int s = h->ctx->find_slot(modulus);
    if (s < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modulus is not part of this context");
    return host_pipeline(h, ntt_op(*h->ctx, h->ctx->map_single(s), data, 1, inverse), rows, Words::u64);
}
int32_t hecuda_ntt_forward_rows(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows) {
    return ntt_rows(h, modulus, data, rows, false);
}
int32_t hecuda_ntt_inverse_rows(const hecuda_context *h, uint64_t modulus, uint64_t *data, int64_t rows) {
    return ntt_rows(h, modulus, data, rows, true);
}

// ---------------------------------------------------------------- multiply

static int32_t bfv_multiply(const hecuda_context *h, const void *lhs, const void *rhs, void *out, int64_t batch, Target t) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (batch < 0 || (batch && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n;
    return run(h,
               {"multiply", {{lhs, in_words}, {rhs, in_words}}, out, (size_t)3 * c.L * c.n, multiply_scratch_words(c), h->chunk,
                h->chunk, [&](const Chunk &x) { return multiply_chunk(c, x.scratch, x.in[0], x.in[1], x.out, x.items, x.stream); }},
               batch, t);
}
int32_t hecuda_bfv_multiply_device(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                   int64_t batch, void *stream) {
    return bfv_multiply(h, lhs, rhs, out, batch, on_stream(stream));
}
int32_t hecuda_bfv_multiply(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                            int64_t batch) {
    return bfv_multiply(h, lhs, rhs, out, batch, kHost64);
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
    if (k->d_block) cudaFree(k->d_block);
    if (k->owns(k->d_relin)) cudaFree(k->d_relin);
    for (auto &kv : k->galois)
        if (k->owns(kv.second)) cudaFree(kv.second);
    for (hecuda::u64 *p : k->retired)
        if (k->owns(p)) cudaFree(p);
    delete k;
    return HECUDA_OK;
}
int32_t hecuda_evk_copy(const hecuda_evk *key, const hecuda_context *h, hecuda_evk **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!key || !key->owner) return fail(HECUDA_ERR_MISSING_KEY, "null evaluation key");
    const Context &a = *key->owner->ctx, &b = *h->ctx;
    // BFV keys do not depend on t: the key is valid wherever N, the word size and every coefficient modulus agree
    if (a.n != b.n || a.word_bits != b.word_bits || a.q != b.q || a.q_ks != b.q_ks)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: the key's context differs in N, word size or coefficient moduli");
    hecuda_evk *k = nullptr;
    if ((rc = hecuda_evk_create_empty(h, &k))) return rc;
    hecuda_evk *src = const_cast<hecuda_evk *>(key);
    cudaError_t e;
    {
        std::lock_guard<std::mutex> lock(src->mu);
        e = cudaMemcpy(k->d_relin, src->d_relin, k->words * sizeof(u64), cudaMemcpyDeviceToDevice);
        for (auto it = src->galois.begin(); e == cudaSuccess && it != src->galois.end(); ++it) {
            u64 *d = nullptr;
            if ((e = cudaMalloc(&d, k->words * sizeof(u64))) != cudaSuccess) break;
            k->galois[it->first] = d;
            e = cudaMemcpy(d, it->second, k->words * sizeof(u64), cudaMemcpyDeviceToDevice);
        }
        k->loaded = src->loaded;
    }
    // the copy is read on other non-blocking streams: publish it once the legacy-stream copies are done (see upload())
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    if (e != cudaSuccess) {
        hecuda_evk_destroy(k);
        return cuda_fail(e, "evk_copy");
    }
    *out = k;
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

// The key checks of the key-switching operations: a key (with its relinearization key when `relin`) made for `h`.
static int32_t check_key(const hecuda_context *h, const hecuda_evk *k, bool relin) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k || (relin && !k->loaded))
        return fail(HECUDA_ERR_MISSING_KEY, relin ? "missingRelinearizationKey" : "missingGaloisKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    return HECUDA_OK;
}
static int32_t check_moduli(const hecuda_context *h, int32_t l) {
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    return HECUDA_OK;
}

static int32_t check_relin(const hecuda_context *h, const hecuda_evk *k, const void *ct3, int32_t l, const void *out,
                           int64_t batch) {
    int32_t rc = check_key(h, k, true);
    if (rc || (rc = check_moduli(h, l))) return rc;
    if (batch < 0 || (batch && (!ct3 || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    return HECUDA_OK;
}

static int32_t bfv_relinearize(const hecuda_context *h, const hecuda_evk *k, const void *ct3, int32_t l, void *out,
                               int64_t batch, Target t) {
    int32_t rc = check_relin(h, k, ct3, l, out, batch);
    if (rc) return rc;
    const Context &c = *h->ctx;
    return run(h,
               {"relinearize", {{ct3, (size_t)3 * l * c.n}}, out, (size_t)2 * l * c.n, relinearize_scratch_words(c, l), h->chunk,
                h->chunk,
                [&](const Chunk &x) { return relinearize_chunk(c, x.scratch, k->d_relin, x.in[0], l, x.out, x.items, x.stream); }},
               batch, t);
}
int32_t hecuda_bfv_relinearize_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                                      uint64_t *out, int64_t batch, void *stream) {
    return bfv_relinearize(h, k, ct3, l, out, batch, on_stream(stream));
}
int32_t hecuda_bfv_relinearize(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                               uint64_t *out, int64_t batch) {
    return bfv_relinearize(h, k, ct3, l, out, batch, kHost64);
}

static int32_t bfv_mod_switch_down(const hecuda_context *h, const void *ct, int32_t polys, int32_t l, void *out, int64_t batch,
                                   Target t) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count");
    if (l < 2 || l > h->ctx->L)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (2 <= moduli_count <= L)");
    if (batch < 0 || (batch && (!ct || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)polys * l * c.n;
    return run(h,
               {"mod_switch", {{ct, in_words}}, out, (size_t)polys * (l - 1) * c.n, 0, kWholeBatch, stage_items(kStageWords, in_words),
                [&](const Chunk &x) { return launch_mod_switch(c, x.in[0], l, x.out, x.items * polys, x.stream); }},
               batch, t);
}
int32_t hecuda_bfv_mod_switch_down_device(const hecuda_context *h, const uint64_t *ct, int32_t polys, int32_t l,
                                          uint64_t *out, int64_t batch, void *stream) {
    return bfv_mod_switch_down(h, ct, polys, l, out, batch, on_stream(stream));
}
int32_t hecuda_bfv_mod_switch_down(const hecuda_context *h, const uint64_t *ct, int32_t polys, int32_t l, uint64_t *out,
                                   int64_t batch) {
    return bfv_mod_switch_down(h, ct, polys, l, out, batch, kHost64);
}

// ---------------------------------------------------------------- relinearize -> modSwitchDown, fused
// Bfv.relinearize then Bfv.modSwitchDown on a batch in one pass (BASELINE config 3): the relinearized ciphertext stays
// in HBM, 2 x (l-1) rows per ciphertext come back.
static int32_t relinearize_mod_switch_down(const hecuda_context *h, const hecuda_evk *k, const void *ct3, int32_t l, void *out,
                                           int64_t batch, Words words) {
    int32_t rc = check_relin(h, k, ct3, l, out, batch);
    if (rc) return rc;
    if (l < 2) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (moduli_count >= 2)");
    const Context &c = *h->ctx;
    const size_t ks_words = relinearize_scratch_words(c, l);
    return host_pipeline(h,
                         {"relinearize_mod_switch_down", {{ct3, (size_t)3 * l * c.n}}, out, (size_t)2 * (l - 1) * c.n,
                          ks_words + (size_t)2 * l * c.n, h->chunk, h->chunk,
                          [&](const Chunk &x) {
                              u64 *relin = x.scratch + ks_words * (size_t)x.items;
                              cudaError_t e = relinearize_chunk(c, x.scratch, k->d_relin, x.in[0], l, relin, x.items, x.stream);
                              if (e != cudaSuccess) return e;
                              return launch_mod_switch(c, relin, l, x.out, x.items * 2, x.stream);
                          }},
                         batch, words);
}
int32_t hecuda_bfv_relinearize_mod_switch_down(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct3, int32_t l,
                                               uint64_t *out, int64_t batch) {
    return relinearize_mod_switch_down(h, k, ct3, l, out, batch, Words::u64);
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
static int32_t bfv_multiply_relinearize(const hecuda_context *h, const hecuda_evk *k, const void *lhs, const void *rhs,
                                        int32_t mod_switch, void *out, int64_t batch, Target t) {
    int32_t rc = check_key(h, k, true);
    if (rc) return rc;
    if (mod_switch && h->ctx->L < 2)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: modSwitchDown needs a next context (L >= 2)");
    if (batch < 0 || (batch && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * (c.L - (mod_switch ? 1 : 0)) * c.n;
    const int64_t chunk = std::max<int64_t>(1, h->chunk / 2);
    return run(h,
               {"multiply_relinearize", {{lhs, in_words}, {rhs, in_words}}, out, out_words, mul_relin_scratch_words(c), chunk, chunk,
                [&](const Chunk &x) {
                    return mul_relin_chunk(c, x.scratch, k->d_relin, x.in[0], x.in[1], mod_switch != 0, x.out, x.items, x.stream);
                }},
               batch, t);
}
int32_t hecuda_bfv_multiply_relinearize_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *lhs,
                                               const uint64_t *rhs, int32_t mod_switch, uint64_t *out, int64_t batch,
                                               void *stream) {
    return bfv_multiply_relinearize(h, k, lhs, rhs, mod_switch, out, batch, on_stream(stream));
}
int32_t hecuda_bfv_multiply_relinearize(const hecuda_context *h, const hecuda_evk *k, const uint64_t *lhs, const uint64_t *rhs,
                                        int32_t mod_switch, uint64_t *out, int64_t batch) {
    return bfv_multiply_relinearize(h, k, lhs, rhs, mod_switch, out, batch, kHost64);
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

// EvaluationKey(deserialize:context:) (SerializedKeys.swift:141-157) with every key ciphertext .seeded, for one client
// or many with one EvaluationKeyConfig.  One DRBG chain pass over every seed of the call, then per group of keys the
// upload of their poly0 bytes and one fused kernel that writes poly0 and poly1 of every ciphertext into the keys'
// device buffers (drbg.cu); groups alternate between two streams, so a group's upload overlaps the previous group's
// expansion.

static int32_t check_key_elements(const Context &c, const uint32_t *elements, int32_t element_count) {
    std::vector<uint32_t> sorted(elements, elements + element_count);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t e : sorted)
        if (!valid_galois_element(e, c.n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element " + std::to_string(e));
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "repeated Galois element " + std::to_string(*std::adjacent_find(sorted.begin(), sorted.end())));
    return HECUDA_OK;
}

// One client's wire bytes as two runs of key ciphertexts: [0] the relinearization key's, [1] the Galois keys'.
// one_buffer: poly0[1] continues poly0[0] in one allocation (a copy must not span two allocations, even adjacent ones).
struct KeyWire {
    const uint8_t *poly0[2], *seeds[2];
    bool one_buffer;
};

// The device side of load_serialized_keys: cts[p] ciphertexts in run p of every client; ciphertext i of client j
// (in the order of its runs) lands at dst[j x per_key + i].
static cudaError_t expand_serialized_keys(const hecuda_context *h, size_t poly_bytes, const int64_t cts[2], int32_t count,
                                          const KeyWire *wire, const std::vector<u64 *> &dst) {
    const Context &c = *h->ctx;
    const int64_t per_key = cts[0] + cts[1], total = per_key * count;
    const size_t key_bytes = poly_bytes * per_key;
    const int32_t group = (int32_t)std::max<uint64_t>(
        1, std::min<uint64_t>(HECUDA_EVK_LOAD_GROUP, HECUDA_EVK_LOAD_GROUP_BYTES / key_bytes));
    std::vector<unsigned char> seeds((size_t)total * 32);
    for (int32_t j = 0; j < count; ++j)
        for (int p = 0; p < 2; ++p)
            if (cts[p]) memcpy(seeds.data() + 32 * (j * per_key + (p ? cts[0] : 0)), wire[j].seeds[p], 32 * (size_t)cts[p]);
    DbStaging st(h);
    if (!st.g0.w || !st.g1.w) return cudaErrorMemoryAllocation;
    const cudaStream_t s0 = st.stream[0];
    const int segments = key_segments(c);
    unsigned char *d_seeds = nullptr;
    u64 **d_dst = nullptr;
    unsigned int *d_rk = nullptr;
    u64 *d_ctr = nullptr;
    cudaEvent_t chained = nullptr;
    cudaError_t e = st.init(key_bytes * std::min(group, count), false);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&chained, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_seeds, seeds.size(), s0);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_dst, sizeof(u64 *) * total, s0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seeds, seeds.data(), seeds.size(), cudaMemcpyHostToDevice, s0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_dst, dst.data(), sizeof(u64 *) * total, cudaMemcpyHostToDevice, s0);
    if (e == cudaSuccess) e = drbg_chains(d_seeds, segments, total, &d_rk, &d_ctr, s0);
    if (e == cudaSuccess) e = cudaEventRecord(chained, s0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st.stream[1], chained, 0);
    for (int32_t first = 0, g = 0; first < count && e == cudaSuccess; first += group, ++g) {
        const int b = g & 1;
        const int32_t keys = std::min(group, count - first);
        // the group's poly0 bytes into st.dev[b], key after key: one copy per client buffer.  A pinned buffer is copied
        // by DMA directly; a pageable one through the driver's pinned staging, which returns once the bytes are staged,
        // so the host moves on to the next group while this group's expansion runs on the other stream.
        for (int32_t j = first; j < first + keys && e == cudaSuccess; ++j) {
            unsigned char *at = st.dev[b] + key_bytes * (j - first);
            if (wire[j].one_buffer) {
                e = cudaMemcpyAsync(at, wire[j].poly0[0], key_bytes, cudaMemcpyHostToDevice, st.stream[b]);
                continue;
            }
            for (int p = 0; p < 2 && e == cudaSuccess; at += poly_bytes * cts[p++])
                if (cts[p]) e = cudaMemcpyAsync(at, wire[j].poly0[p], poly_bytes * cts[p], cudaMemcpyHostToDevice, st.stream[b]);
        }
        if (e == cudaSuccess)
            e = expand_key_ciphertexts(c, d_rk, d_ctr, first * per_key, keys * per_key, st.dev[b], d_dst, st.stream[b]);
    }
    // the chains are zeroized and freed once both streams' expansions have read them; the keys are read on other
    // non-blocking streams, so return once they are written (see upload())
    cudaError_t e2 = wait_stream(st.stream[1]);
    if (e == cudaSuccess) e = e2;
    free_chains(d_rk, d_ctr, segments, total, s0);
    for (void *p : {(void *)d_seeds, (void *)d_dst})
        if (p) cudaFreeAsync(p, s0);
    e2 = wait_stream(s0);
    if (e == cudaSuccess) e = e2;
    if (chained) cudaEventDestroy(chained);
    return e;
}

// SerializedEvaluationKey messages, walked (pirproto::walk_evaluation_key): every message goes to the device as it is,
// one DRBG chain launch covers every seed and one expansion launch every ciphertext, both reading them in place.
// Ciphertext i of client j in message order lands at dst[j x per_key + canonical index] (the relinearization key, then
// elements[] in order).
struct KeyMessages {
    const uint8_t *const *messages;
    const uint64_t *byte_counts;
    std::vector<pirproto::EvaluationKey> keys;
};

static cudaError_t expand_proto_keys(const hecuda_context *h, const KeyMessages &km, const uint32_t *elements,
                                     int32_t element_count, bool relin, const std::vector<u64 *> &dst) {
    const Context &c = *h->ctx;
    const int32_t count = (int32_t)km.keys.size();
    const int64_t per_key = (int64_t)(relin ? c.L : 0) + (int64_t)element_count * c.L, total = per_key * count;
    std::vector<u64 *> ordered((size_t)total);
    std::vector<long long> tables((size_t)total * 2);  // poly0 offsets, then seed offsets, into the uploaded messages
    size_t bytes = 0;
    for (int32_t j = 0; j < count; ++j) {
        const pirproto::EvaluationKey &k = km.keys[(size_t)j];
        for (size_t m = 0; m < k.order.size(); ++m) {
            const int key = k.order[m].first, i = k.order[m].second;
            const pirproto::Ciphertext &ct = key < 0 ? k.relin_cts[(size_t)i] : k.galois[(size_t)key].cts[(size_t)i];
            int64_t canonical = i;
            if (key >= 0) {
                const int32_t g = (int32_t)(std::find(elements, elements + element_count, (uint32_t)k.galois[(size_t)key].element) - elements);
                canonical = (relin ? c.L : 0) + (int64_t)g * c.L + i;
            }
            const size_t at = (size_t)(j * per_key) + m;
            ordered[at] = dst[(size_t)(j * per_key + canonical)];
            tables[at] = (long long)bytes + ct.poly[0];
            tables[(size_t)total + at] = (long long)bytes + ct.seed;
        }
        bytes += km.byte_counts[j];
    }
    WsGuard g(h);
    if (!g.w) return cudaErrorMemoryAllocation;
    const cudaStream_t s = g.w->stream;
    const int segments = key_segments(c);
    unsigned char *d_msg = nullptr;
    long long *d_tables = nullptr;
    u64 **d_dst = nullptr;
    unsigned int *d_rk = nullptr;
    u64 *d_ctr = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_msg, std::max<size_t>(bytes, 1), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_tables, tables.size() * sizeof(long long), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_dst, sizeof(u64 *) * total, s);
    // each message is one copy: by DMA directly when it is pinned, through the driver's pinned staging when pageable
    for (size_t j = 0, offset = 0; j < (size_t)count && e == cudaSuccess; offset += km.byte_counts[j++])
        e = cudaMemcpyAsync(d_msg + offset, km.messages[j], km.byte_counts[j], cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_tables, tables.data(), tables.size() * sizeof(long long), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_dst, ordered.data(), sizeof(u64 *) * total, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = drbg_chains(d_msg, segments, total, &d_rk, &d_ctr, s, d_tables + total);
    PolyLayout at;
    at.tag = d_tables, at.frame = 0;
    if (e == cudaSuccess) e = expand_key_ciphertexts(c, d_rk, d_ctr, 0, total, d_msg, d_dst, s, at);
    free_chains(d_rk, d_ctr, segments, total, s);
    for (void *p : {(void *)d_msg, (void *)d_tables, (void *)d_dst})
        if (p) cudaFreeAsync(p, s);
    const cudaError_t e2 = wait_stream(s);
    return e == cudaSuccess ? e2 : e;
}

// `count` clients' keys of one config, every argument already checked: one allocation per key, then the expansion
// (of the wire arrays, or of the messages `km`).  On error nothing is left allocated and out[] is untouched.
static int32_t load_serialized_keys(const hecuda_context *h, uint64_t poly_bytes, int32_t count, bool relin,
                                    const uint32_t *elements, int32_t element_count, const KeyWire *wire, hecuda_evk **out,
                                    const KeyMessages *km = nullptr) {
    const Context &c = *h->ctx;
    const size_t words = (size_t)c.L * 2 * (c.L + 1) * c.n, ct_words = words / c.L;
    const int64_t cts[2] = {relin ? c.L : 0, (int64_t)element_count * c.L};
    std::vector<hecuda_evk *> keys;
    // ciphertext i of a key lands at key + i x 2 x K x N: its relinearization key, then galois[elements[e]]
    std::vector<u64 *> dst;
    dst.reserve((size_t)(cts[0] + cts[1]) * count);
    cudaError_t e = cudaSuccess;
    for (int32_t j = 0; j < count && e == cudaSuccess; ++j) {
        hecuda_evk *k = new (std::nothrow) hecuda_evk();
        if (!k) {
            e = cudaErrorMemoryAllocation;
            break;
        }
        keys.push_back(k);
        k->owner = h;
        k->words = words;
        k->block_words = words * (1 + (size_t)element_count);  // d_relin is allocated even without a relinearization key
        if ((e = cudaMalloc(&k->d_block, k->block_words * sizeof(u64))) != cudaSuccess) break;
        k->d_relin = k->d_block;
        for (int32_t g = relin ? -1 : 0; g < element_count; ++g) {
            u64 *key = k->d_block + words * (1 + g);
            if (g >= 0) k->galois[elements[g]] = key;
            for (int i = 0; i < c.L; ++i) dst.push_back(key + ct_words * i);
        }
        k->loaded = relin;
    }
    if (e == cudaSuccess && !dst.empty())
        e = km ? expand_proto_keys(h, *km, elements, element_count, relin, dst)
               : expand_serialized_keys(h, (size_t)poly_bytes, cts, count, wire, dst);
    if (e != cudaSuccess) {
        for (hecuda_evk *k : keys) hecuda_evk_destroy(k);
        return cuda_fail(e, "evk_create_serialized");
    }
    std::copy(keys.begin(), keys.end(), out);
    return HECUDA_OK;
}

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
    if ((rc = check_key_elements(c, elements, element_count))) return rc;
    uint64_t poly_bytes = 0;
    if ((rc = hecuda_poly_serialized_byte_count(h, HECUDA_BASE_KEYSWITCH, c.L + 1, 0, &poly_bytes))) return rc;
    const KeyWire wire{{relin_poly0, galois_poly0}, {relin_seeds, galois_seeds}, false};
    return load_serialized_keys(h, poly_bytes, 1, relin_poly0 != nullptr, elements, element_count, &wire, out);
}

int32_t hecuda_evk_create_serialized_many(const hecuda_context *h, int32_t key_count, int32_t has_relin,
                                          const uint32_t *elements, int32_t element_count, const uint8_t *const *poly0,
                                          const uint8_t *const *seeds, hecuda_evk **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (key_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "key_count " + std::to_string(key_count) + ": expected at least 1");
    std::fill(out, out + key_count, nullptr);
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!c.has_ks)
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: a single coefficient modulus leaves no key-switching modulus");
    if (element_count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "element_count " + std::to_string(element_count) + " < 0");
    if (element_count > 0 && !elements) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if ((rc = check_key_elements(c, elements, element_count))) return rc;
    uint64_t poly_bytes = 0;
    if ((rc = hecuda_poly_serialized_byte_count(h, HECUDA_BASE_KEYSWITCH, c.L + 1, 0, &poly_bytes))) return rc;
    const bool relin = has_relin != 0;
    const bool any = relin || element_count > 0;
    if (any && (!poly0 || !seeds)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const size_t relin_cts = relin ? (size_t)c.L : 0;
    std::vector<KeyWire> wire((size_t)key_count, KeyWire{{nullptr, nullptr}, {nullptr, nullptr}, true});
    for (int32_t j = 0; any && j < key_count; ++j) {
        if (!poly0[j] || !seeds[j]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "client " + std::to_string(j) + ": null argument");
        wire[(size_t)j] = KeyWire{{poly0[j], poly0[j] + poly_bytes * relin_cts}, {seeds[j], seeds[j] + 32 * relin_cts}, true};
    }
    return load_serialized_keys(h, poly_bytes, key_count, relin, elements, element_count, wire.data(), out);
}

int32_t hecuda_evk_create_proto_many(const hecuda_context *h, int32_t key_count, const uint8_t *const *messages,
                                     const uint64_t *message_byte_counts, hecuda_evk **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (key_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "key_count " + std::to_string(key_count) + ": expected at least 1");
    std::fill(out, out + key_count, nullptr);
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!c.has_ks)
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: a single coefficient modulus leaves no key-switching modulus");
    if (!messages || !message_byte_counts) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    CodecConsts cc;
    std::string err;
    if (!codec_consts(c, c.map_ks(c.L), 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const pirproto::PolySizes sz = pirproto::poly_sizes(cc, c.n);
    KeyMessages km{messages, message_byte_counts, std::vector<pirproto::EvaluationKey>((size_t)key_count)};
    std::vector<uint32_t> elements, sorted;
    for (int32_t j = 0; j < key_count; ++j) {
        const std::string who = "client " + std::to_string(j) + ": ";
        if (!messages[j]) return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "null argument");
        pirproto::Error e;
        pirproto::EvaluationKey &k = km.keys[(size_t)j];
        if (!pirproto::walk_evaluation_key(messages[j], 0, (long long)message_byte_counts[j], sz, c.L, k, e))
            return fail(e.code, who + e.what);
        std::vector<uint32_t> mine;
        for (const pirproto::GaloisKey &gk : k.galois) {
            if (gk.element > 0xffffffffull || !valid_galois_element((uint32_t)gk.element, c.n))
                return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "invalid Galois element " + std::to_string(gk.element));
            mine.push_back((uint32_t)gk.element);
        }
        if (j == 0) {
            elements = mine;  // the call's configuration: client 0's elements, in its map order
            sorted = mine;
            std::sort(sorted.begin(), sorted.end());
            continue;
        }
        if (k.relin != km.keys[0].relin)
            return fail(HECUDA_ERR_INVALID_ARGUMENT,
                        who + "relinearization key " + (k.relin ? "present" : "absent") + ", unlike client 0");
        std::sort(mine.begin(), mine.end());
        if (mine != sorted) return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "Galois elements differ from client 0's");
    }
    uint64_t poly_bytes = 0;
    if ((rc = hecuda_poly_serialized_byte_count(h, HECUDA_BASE_KEYSWITCH, c.L + 1, 0, &poly_bytes))) return rc;
    return load_serialized_keys(h, poly_bytes, key_count, km.keys[0].relin, elements.data(), (int32_t)elements.size(),
                                nullptr, out, &km);
}

static int32_t bfv_apply_galois(const hecuda_context *h, const hecuda_evk *k, const void *ct, int32_t l, uint32_t element,
                                void *out, int64_t batch, Target t) {
    int32_t rc = check_key(h, k, false);
    if (rc) return rc;
    if (!valid_galois_element(element, h->ctx->n)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element");
    if ((rc = check_moduli(h, l))) return rc;
    if (batch < 0 || (batch && (!ct || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const u64 *key = nullptr;
    {
        hecuda_evk *km = const_cast<hecuda_evk *>(k);
        std::lock_guard<std::mutex> g(km->mu);
        auto it = km->galois.find(element);
        if (it == km->galois.end()) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisElement: " + std::to_string(element));
        key = it->second;
    }
    const Context &c = *h->ctx;
    const size_t words = (size_t)2 * l * c.n;
    return run(h,
               {"applyGalois", {{ct, words}}, out, words, galois_scratch_words(c, l), h->chunk, h->chunk,
                [&](const Chunk &x) { return apply_galois_chunk(c, x.scratch, key, x.in[0], l, element, x.out, x.items, x.stream); }},
               batch, t);
}
int32_t hecuda_bfv_apply_galois_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct, int32_t l,
                                       uint32_t element, uint64_t *out, int64_t batch, void *stream) {
    return bfv_apply_galois(h, k, ct, l, element, out, batch, on_stream(stream));
}
int32_t hecuda_bfv_apply_galois(const hecuda_context *h, const hecuda_evk *k, const uint64_t *ct, int32_t l,
                                uint32_t element, uint64_t *out, int64_t batch) {
    return bfv_apply_galois(h, k, ct, l, element, out, batch, kHost64);
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
    return host_pipeline(h,
                         {"poly_apply_galois", {{in, words}}, out, words, 0, kWholeBatch, stage_items(kStageWords, words),
                          [&](const Chunk &x) {
                              return eval_format ? launch_galois_eval(c, rows, element, x.in[0], x.out, x.items, x.stream)
                                                 : launch_galois_coeff(c, map, element, x.in[0], (int64_t)words, x.out,
                                                                       (int64_t)words, x.items, x.stream);
                          }},
                         polys, Words::u64);
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

// the query ciphertexts `cts` and the presence flags are device buffers here, shared by every output row
static Batched inner_product_plaintexts_op(const Context &c, const u64 *cts, int32_t polys, int32_t l, int64_t terms,
                                           const void *pts, const unsigned char *present, void *out) {
    const size_t pt_words = (size_t)terms * l * c.n;
    return {"inner_product", {{pts, pt_words}}, out, (size_t)polys * l * c.n, 0, kWholeBatch,
            stage_items(8 * kStageWords, pt_words), [&c, cts, polys, l, terms, present](const Chunk &x) {
                return launch_inner_product_plain(c, cts, polys, l, terms, x.in[0], present ? present + x.first * terms : nullptr,
                                                  x.out, x.items, x.stream);
            }};
}
int32_t hecuda_bfv_inner_product_plaintexts_device(const hecuda_context *h, const uint64_t *cts, int32_t polys,
                                                   int32_t l, int64_t terms, const uint64_t *pts,
                                                   const uint8_t *present, uint64_t *out, int64_t out_count,
                                                   void *stream) {
    int32_t rc = check_ip(h, cts, polys, l, terms, pts, out, out_count);
    if (rc) return rc;
    return run_device(inner_product_plaintexts_op(*h->ctx, (const u64 *)cts, polys, l, terms, pts, present, out), out_count,
                      (cudaStream_t)stream);
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
    rc = host_pipeline(h, inner_product_plaintexts_op(c, d_cts, polys, l, terms, pts, d_present, out), out_count, Words::u64);
    cudaFree(d_cts);
    cudaFree(d_present);
    return rc;
}

static int32_t plaintext_to_eval(const hecuda_context *h, const void *plain, int32_t l, void *out, int64_t count, Target t) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count out of range");
    if (count < 0 || (count && (!plain || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    const Context &c = *h->ctx;
    const size_t out_words = (size_t)l * c.n;
    return run(h,
               {"plaintext_to_eval", {{plain, (size_t)c.n}}, out, out_words, 0, kWholeBatch, stage_items(kStageWords, out_words),
                [&](const Chunk &x) { return launch_plaintext_to_eval(c, x.in[0], l, x.out, x.items, x.stream); }},
               count, t);
}
int32_t hecuda_plaintext_to_eval_device(const hecuda_context *h, const uint64_t *plain, int32_t l, uint64_t *out,
                                        int64_t count, void *stream) {
    return plaintext_to_eval(h, plain, l, out, count, on_stream(stream));
}
int32_t hecuda_plaintext_to_eval(const hecuda_context *h, const uint64_t *plain, int32_t l, uint64_t *out,
                                 int64_t count) {
    return plaintext_to_eval(h, plain, l, out, count, kHost64);
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

// encodingDataOutOfBounds (Encoding.swift:147-156) on host buffers
bool host_values_below(const void *p, size_t count, u64 t, Words words) {
    if (words == Words::u32) {
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

static int32_t bfv_encode_simd(const hecuda_context *h, const void *values, int32_t value_count, int32_t l, void *out,
                               int64_t count, Target t) {
    int32_t rc = check_encode(h, values, value_count, l, out, count);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!t.device && !host_values_below(values, (size_t)count * value_count, c.t, t.words))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "encodingDataOutOfBounds: values must be below the plaintext modulus");
    std::vector<Batched::Io> in;
    if (value_count) in.push_back({values, (size_t)value_count});
    const size_t out_words = (size_t)(l ? l : 1) * c.n;
    return run(h,
               {"encodeSimd", in, out, out_words, simd_scratch_words(c, true, l), simd_chunk(c), stage_items(kStageWords, out_words),
                [&](const Chunk &x) {
                    return launch_encode_simd(c, value_count ? x.in[0] : nullptr, value_count, l, x.out, x.scratch, x.items, x.stream);
                }},
               count, t);
}
int32_t hecuda_bfv_encode_simd_device(const hecuda_context *h, const uint64_t *values, int32_t value_count,
                                      int32_t moduli_count, uint64_t *out, int64_t count, void *stream) {
    return bfv_encode_simd(h, values, value_count, moduli_count, out, count, on_stream(stream));
}
int32_t hecuda_bfv_encode_simd(const hecuda_context *h, const uint64_t *values, int32_t value_count, int32_t moduli_count,
                               uint64_t *out, int64_t count) {
    return bfv_encode_simd(h, values, value_count, moduli_count, out, count, kHost64);
}

static int32_t bfv_decode_simd(const hecuda_context *h, const void *plaintexts, int32_t l, void *values, int64_t count,
                               Target t) {
    int32_t rc = check_decode(h, plaintexts, l, values, count);
    if (rc) return rc;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)(l ? l : 1) * c.n;
    return run(h,
               {"decodeSimd", {{plaintexts, in_words}}, values, (size_t)c.n, simd_scratch_words(c, false, l), simd_chunk(c),
                stage_items(kStageWords, in_words),
                [&](const Chunk &x) { return launch_decode_simd(c, x.in[0], l, x.out, x.scratch, x.items, x.stream); }},
               count, t);
}
int32_t hecuda_bfv_decode_simd_device(const hecuda_context *h, const uint64_t *plaintexts, int32_t moduli_count,
                                      uint64_t *values, int64_t count, void *stream) {
    return bfv_decode_simd(h, plaintexts, moduli_count, values, count, on_stream(stream));
}
int32_t hecuda_bfv_decode_simd(const hecuda_context *h, const uint64_t *plaintexts, int32_t moduli_count, uint64_t *values,
                               int64_t count) {
    return bfv_decode_simd(h, plaintexts, moduli_count, values, count, kHost64);
}

static int32_t bfv_plaintext_translate(const hecuda_context *h, const void *ct, int32_t poly_count, int32_t l,
                                       const void *plaintexts, int64_t plaintext_count, int32_t op, void *out, int64_t batch,
                                       Target t) {
    int32_t rc = check_translate(h, ct, poly_count, l, plaintexts, plaintext_count, op, out, batch);
    if (rc || batch == 0) return rc;
    const Context &c = *h->ctx;
    const bool broadcast = plaintext_count == 1;
    const size_t ct_words = (size_t)poly_count * l * c.n;
    std::vector<Batched::Io> in = {{ct, ct_words}};
    const u64 *pt = static_cast<const u64 *>(plaintexts);  // the shared plaintext of a broadcast, on the device
    u64 *d_pt = nullptr;
    if (!t.device) {
        if (!host_values_below(plaintexts, (size_t)plaintext_count * c.n, c.t, t.words))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "encodingDataOutOfBounds: plaintext coefficients must be below t");
        if (broadcast) {  // uploaded once
            std::vector<u64> wide(c.n);
            if (t.words == Words::u32) std::copy((const uint32_t *)plaintexts, (const uint32_t *)plaintexts + c.n, wide.begin());
            else std::copy(pt, pt + c.n, wide.begin());
            CK(cudaMalloc(&d_pt, sizeof(u64) * (size_t)c.n));
            cudaError_t e = upload(d_pt, wide.data(), sizeof(u64) * (size_t)c.n);
            if (e != cudaSuccess) {
                cudaFree(d_pt);
                return cuda_fail(e, "plaintext upload");
            }
            pt = d_pt;
        }
    }
    if (!broadcast) in.push_back({plaintexts, (size_t)c.n});
    rc = run(h,
             {"plaintextTranslate", in, out, ct_words, 0, kWholeBatch, stage_items(kStageWords, ct_words),
              [&](const Chunk &x) {
                  return launch_plaintext_translate(c, x.in[0], poly_count, l, broadcast ? pt : x.in[1], broadcast, op, x.out,
                                                    x.items, x.stream);
              }},
             batch, t);
    if (d_pt) cudaFree(d_pt);
    return rc;
}
int32_t hecuda_bfv_plaintext_translate_device(const hecuda_context *h, const uint64_t *ct, int32_t poly_count,
                                              int32_t moduli_count, const uint64_t *plaintexts, int64_t plaintext_count,
                                              int32_t op, uint64_t *out, int64_t batch, void *stream) {
    return bfv_plaintext_translate(h, ct, poly_count, moduli_count, plaintexts, plaintext_count, op, out, batch,
                                   on_stream(stream));
}
int32_t hecuda_bfv_plaintext_translate(const hecuda_context *h, const uint64_t *ct, int32_t poly_count, int32_t moduli_count,
                                       const uint64_t *plaintexts, int64_t plaintext_count, int32_t op, uint64_t *out,
                                       int64_t batch) {
    return bfv_plaintext_translate(h, ct, poly_count, moduli_count, plaintexts, plaintext_count, op, out, batch, kHost64);
}

// ---------------------------------------------------------------- ct x ct inner product (SURVEY.md 8f rank 2)

static int32_t check_ipc(const hecuda_context *h, const void *lhs, const void *rhs, const void *out, int64_t pairs,
                         int64_t groups) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (pairs < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "Empty ciphertexts");
    if (groups < 0 || (groups && (!lhs || !rhs || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    if (h->ctx->n < 2) return fail(HECUDA_ERR_UNSUPPORTED, "degree too small");
    return HECUDA_OK;
}

static int32_t bfv_inner_product(const hecuda_context *h, const void *lhs, const void *rhs, void *out, int64_t pairs,
                                 int64_t groups, Target t) {
    int32_t rc = check_ipc(h, lhs, rhs, out, pairs, groups);
    if (rc) return rc;
    const Context &c = *h->ctx;
    const size_t in_words = (size_t)pairs * 2 * c.L * c.n;
    const int64_t chunk = std::max<int64_t>(1, h->chunk / pairs);  // groups
    return run(h,
               {"innerProduct", {{lhs, in_words}, {rhs, in_words}}, out, (size_t)3 * c.L * c.n, inner_product_scratch_words(c, pairs),
                chunk, chunk,
                [&](const Chunk &x) { return inner_product_chunk(c, x.scratch, x.in[0], x.in[1], pairs, x.out, x.items, x.stream); }},
               groups, t);
}
int32_t hecuda_bfv_inner_product_device(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                        int64_t pairs, int64_t groups, void *stream) {
    return bfv_inner_product(h, lhs, rhs, out, pairs, groups, on_stream(stream));
}
int32_t hecuda_bfv_inner_product(const hecuda_context *h, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                 int64_t pairs, int64_t groups) {
    return bfv_inner_product(h, lhs, rhs, out, pairs, groups, kHost64);
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
    return host_pipeline(h,
                         {"multiply_power_of_x", {{in, words}}, out, words, 0, kWholeBatch, stage_items(kStageWords, words),
                          [&](const Chunk &x) { return launch_multiply_power_of_x(c, map, power, x.in[0], x.out, x.items, x.stream); }},
                         polys, Words::u64);
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
    return rc ? rc : ntt(h, base, data, rows, polys, false, kHost32);
}
int32_t hecuda_u32_ntt_inverse(const hecuda_context *h, int32_t base, uint32_t *data, int32_t rows, int64_t polys) {
    int32_t rc = need_word32(h);
    return rc ? rc : ntt(h, base, data, rows, polys, true, kHost32);
}
int32_t hecuda_u32_bfv_multiply(const hecuda_context *h, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_multiply(h, lhs, rhs, out, batch, kHost32);
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
    return rc ? rc : bfv_relinearize(h, evk, ct3, l, out, batch, kHost32);
}
int32_t hecuda_u32_bfv_mod_switch_down(const hecuda_context *h, const uint32_t *ct, int32_t polys, int32_t l, uint32_t *out,
                                       int64_t batch) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_mod_switch_down(h, ct, polys, l, out, batch, kHost32);
}
int32_t hecuda_u32_bfv_multiply_relinearize(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *lhs, const uint32_t *rhs,
                                            int32_t mod_switch, uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_multiply_relinearize(h, evk, lhs, rhs, mod_switch, out, batch, kHost32);
}
int32_t hecuda_u32_bfv_relinearize_mod_switch_down(const hecuda_context *h, const hecuda_evk *evk, const uint32_t *ct3, int32_t l,
                                                   uint32_t *out, int64_t batch) {
    int32_t rc = need_word32(h);
    return rc ? rc : relinearize_mod_switch_down(h, evk, ct3, l, out, batch, Words::u32);
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
    return rc ? rc : bfv_apply_galois(h, evk, ct, l, element, out, batch, kHost32);
}
int32_t hecuda_u32_bfv_inner_product(const hecuda_context *h, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out, int64_t pairs,
                                     int64_t groups) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_inner_product(h, lhs, rhs, out, pairs, groups, kHost32);
}
int32_t hecuda_u32_rnstool_lift_q_to_qbsk(const hecuda_context *h, const uint32_t *polys, uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    return rc ? rc : lift_or_floor(h, polys, out, count, true, Words::u32);
}
int32_t hecuda_u32_rnstool_floor_qbsk_to_q(const hecuda_context *h, const uint32_t *polys, uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    return rc ? rc : lift_or_floor(h, polys, out, count, false, Words::u32);
}
int32_t hecuda_u32_bfv_encode_simd(const hecuda_context *h, const uint32_t *values, int32_t value_count, int32_t moduli_count,
                                   uint32_t *out, int64_t count) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_encode_simd(h, values, value_count, moduli_count, out, count, kHost32);
}
int32_t hecuda_u32_bfv_decode_simd(const hecuda_context *h, const uint32_t *plaintexts, int32_t moduli_count, uint32_t *values,
                                   int64_t count) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_decode_simd(h, plaintexts, moduli_count, values, count, kHost32);
}
int32_t hecuda_u32_bfv_plaintext_translate(const hecuda_context *h, const uint32_t *ct, int32_t poly_count, int32_t moduli_count,
                                           const uint32_t *plaintexts, int64_t plaintext_count, int32_t op, uint32_t *out,
                                           int64_t batch) {
    int32_t rc = need_word32(h);
    return rc ? rc : bfv_plaintext_translate(h, ct, poly_count, moduli_count, plaintexts, plaintext_count, op, out, batch, kHost32);
}

}  // extern "C"
