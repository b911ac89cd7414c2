// elementwise.cu -- coefficient-wise PolyRq arithmetic (SURVEY.md 8a row a7).
//
//   PolyRq += / -=                  PolyRq/PolyRq.swift:147-174
//   PolyRq *= PolyRq (Eval format)  PolyRq/PolyRq.swift:184-204   (Modulus.multiplyMod, Modulus.swift:89-94)
//   -PolyRq                         PolyRq/PolyRq.swift (negation, negateMod Scalar.swift:167-175)
//   PolyRq *= [T]                   PolyRq/PolyRq.swift:232-245   (one scalar per RNS row)
//
// The fused kernels of the hot path never materialise these steps; the entry points exist so that a caller that keeps
// ciphertexts resident in HBM (Ciphertext += Ciphertext, Ciphertext *= Plaintext, ...) does not have to leave the device.
// All are HBM-bound streaming kernels: thread = two adjacent coefficients, 16-byte accesses.
#include "capi_internal.hpp"
#include "modarith.cuh"

using namespace hecuda;
using namespace hecuda::api;

namespace {

enum { kAdd = 0, kSub = 1, kMul = 2, kNeg = 3, kScalar = 4 };

struct EwConsts {
    int rows;
    u64 p[kMaxRows], mu_hi[kMaxRows], mu_lo[kMaxRows];
    u64 scalar[kMaxRows];  // kScalar only
};

template <int OP>
__device__ __forceinline__ u64 apply(u64 a, u64 b, u64 p, u64 mu_hi, u64 mu_lo) {
    if (OP == kAdd) return add_mod(a, b, p);
    if (OP == kSub) return sub_mod(a, b, p);
    if (OP == kNeg) return a ? p - a : 0;
    return barrett128(mul_wide(a, b), p, mu_hi, mu_lo);  // kMul, kScalar
}

template <int OP>
__global__ void __launch_bounds__(256) elementwise_kernel(u64 *__restrict__ lhs, const u64 *__restrict__ rhs,
                                                         const __grid_constant__ EwConsts c, int n) {
    const int e = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (e >= n) return;
    const int row = blockIdx.y;
    const int64_t off = ((int64_t)blockIdx.z * c.rows + row) * n + e;
    const u64 p = c.p[row], mu_hi = c.mu_hi[row], mu_lo = c.mu_lo[row];
    if (e + 1 < n) {
        ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(lhs + off);
        ulonglong2 b = make_ulonglong2(c.scalar[row], c.scalar[row]);
        if (OP == kAdd || OP == kSub || OP == kMul) b = *reinterpret_cast<const ulonglong2 *>(rhs + off);
        a.x = apply<OP>(a.x, b.x, p, mu_hi, mu_lo);
        a.y = apply<OP>(a.y, b.y, p, mu_hi, mu_lo);
        *reinterpret_cast<ulonglong2 *>(lhs + off) = a;
    } else {  // N = 1
        const u64 b = (OP == kAdd || OP == kSub || OP == kMul) ? rhs[off] : c.scalar[row];
        lhs[off] = apply<OP>(lhs[off], b, p, mu_hi, mu_lo);
    }
}

cudaError_t launch_elementwise(const Context &ctx, const NttRowMap &map, int op, u64 *lhs, const u64 *rhs, const u64 *scalars,
                               int64_t polys, cudaStream_t s) {
    if (polys == 0) return cudaSuccess;
    EwConsts c;
    c.rows = map.rows_per_poly;
    for (int r = 0; r < c.rows; ++r) {
        const ModSlot &S = ctx.slots[map.slot[r]].dev;
        c.p[r] = S.p;
        c.mu_hi[r] = S.mu_hi;
        c.mu_lo[r] = S.mu_lo;
        c.scalar[r] = scalars ? scalars[r] : 0;
    }
    const int threads = coeff_threads(ctx.n / 2);
    const unsigned gx = (unsigned)(((ctx.n + 1) / 2 + threads - 1) / threads);
    auto kernel = op == kAdd ? elementwise_kernel<kAdd>
                : op == kSub ? elementwise_kernel<kSub>
                : op == kMul ? elementwise_kernel<kMul>
                : op == kNeg ? elementwise_kernel<kNeg>
                             : elementwise_kernel<kScalar>;
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid(gx, (unsigned)c.rows, (unsigned)chunk);
        return launch(kernel, grid, threads, 0, s, lhs + done * c.rows * ctx.n, rhs ? rhs + done * c.rows * ctx.n : nullptr, c,
                      (int)ctx.n);
    });
}

int32_t run(const hecuda_context *h, int32_t base, int op, uint64_t *lhs, const uint64_t *rhs, const uint64_t *scalars,
            int32_t rows, int64_t polys, bool device, void *stream) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    const bool binary = op == kAdd || op == kSub || op == kMul;
    if (polys < 0 || (polys && (!lhs || (binary && !rhs)))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid data / poly_count");
    if (op == kScalar && !scalars) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null scalars");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const Context &c = *h->ctx;
    if (op == kScalar)
        for (int r = 0; r < rows; ++r)
            if (scalars[r] >= c.slots[map.slot[r]].dev.p) return fail(HECUDA_ERR_INVALID_ARGUMENT, "scalar not reduced modulo its row modulus");
    if (polys == 0) return HECUDA_OK;
    if (device) {
        cudaError_t e = launch_elementwise(c, map, op, (u64 *)lhs, (const u64 *)rhs, (const u64 *)scalars, polys, (cudaStream_t)stream);
        return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "elementwise");
    }
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    const size_t words = (size_t)rows * c.n;
    const int64_t slab = std::max<int64_t>(1, (int64_t)((size_t)32 * 1024 * 1024 / words));
    u64 *d_l = nullptr, *d_r = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_l, words * std::min(slab, polys) * sizeof(u64), s);
    if (e == cudaSuccess && binary) e = cudaMallocAsync((void **)&d_r, words * std::min(slab, polys) * sizeof(u64), s);
    for (int64_t done = 0; e == cudaSuccess && done < polys; done += slab) {
        const int64_t items = std::min(slab, polys - done);
        e = cudaMemcpyAsync(d_l, lhs + words * done, words * items * sizeof(u64), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && binary)
            e = cudaMemcpyAsync(d_r, rhs + words * done, words * items * sizeof(u64), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = launch_elementwise(c, map, op, d_l, d_r, (const u64 *)scalars, items, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(lhs + words * done, d_l, words * items * sizeof(u64), cudaMemcpyDeviceToHost, s);
    }
    if (d_l) cudaFreeAsync(d_l, s);
    if (d_r) cudaFreeAsync(d_r, s);
    cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "elementwise");
}

}  // namespace

extern "C" {

int32_t hecuda_poly_add(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows, int64_t polys) {
    return run(h, base, kAdd, lhs, rhs, nullptr, rows, polys, false, nullptr);
}
int32_t hecuda_poly_sub(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows, int64_t polys) {
    return run(h, base, kSub, lhs, rhs, nullptr, rows, polys, false, nullptr);
}
int32_t hecuda_poly_mul(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows, int64_t polys) {
    return run(h, base, kMul, lhs, rhs, nullptr, rows, polys, false, nullptr);
}
int32_t hecuda_poly_neg(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys) {
    return run(h, base, kNeg, data, nullptr, nullptr, rows, polys, false, nullptr);
}
int32_t hecuda_poly_mul_scalars(const hecuda_context *h, int32_t base, uint64_t *data, const uint64_t *scalars, int32_t rows,
                                int64_t polys) {
    return run(h, base, kScalar, data, nullptr, scalars, rows, polys, false, nullptr);
}
int32_t hecuda_poly_add_device(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows,
                               int64_t polys, void *stream) {
    return run(h, base, kAdd, lhs, rhs, nullptr, rows, polys, true, stream);
}
int32_t hecuda_poly_sub_device(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows,
                               int64_t polys, void *stream) {
    return run(h, base, kSub, lhs, rhs, nullptr, rows, polys, true, stream);
}
int32_t hecuda_poly_mul_device(const hecuda_context *h, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t rows,
                               int64_t polys, void *stream) {
    return run(h, base, kMul, lhs, rhs, nullptr, rows, polys, true, stream);
}
int32_t hecuda_poly_neg_device(const hecuda_context *h, int32_t base, uint64_t *data, int32_t rows, int64_t polys, void *stream) {
    return run(h, base, kNeg, data, nullptr, nullptr, rows, polys, true, stream);
}
int32_t hecuda_poly_mul_scalars_device(const hecuda_context *h, int32_t base, uint64_t *data, const uint64_t *scalars,
                                       int32_t rows, int64_t polys, void *stream) {
    return run(h, base, kScalar, data, nullptr, scalars, rows, polys, true, stream);
}

}  // extern "C"

// ---- word-size conversion at the boundary of a Bfv<UInt32> context: residues travel as uint32 (half the PCIe bytes)
// and sit zero-extended in 64-bit slots on the device.
namespace hecuda {

__global__ void __launch_bounds__(256) widen_kernel(const u32 *__restrict__ in, u64 *__restrict__ out, int64_t words) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < words) {
        const uint4 v = *reinterpret_cast<const uint4 *>(in + i);
        reinterpret_cast<ulonglong2 *>(out + i)[0] = make_ulonglong2(v.x, v.y);
        reinterpret_cast<ulonglong2 *>(out + i)[1] = make_ulonglong2(v.z, v.w);
    } else {
        for (int64_t k = i; k < words; ++k) out[k] = in[k];
    }
}
__global__ void __launch_bounds__(256) narrow_kernel(const u64 *__restrict__ in, u32 *__restrict__ out, int64_t words) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < words) {
        const ulonglong2 a = reinterpret_cast<const ulonglong2 *>(in + i)[0], b = reinterpret_cast<const ulonglong2 *>(in + i)[1];
        *reinterpret_cast<uint4 *>(out + i) = make_uint4((u32)a.x, (u32)a.y, (u32)b.x, (u32)b.y);
    } else {
        for (int64_t k = i; k < words; ++k) out[k] = (u32)in[k];
    }
}
cudaError_t launch_widen(const u32 *in, u64 *out, int64_t words, cudaStream_t stream) {
    if (words == 0) return cudaSuccess;
    return launch(widen_kernel, (unsigned)((words + 1023) / 1024), 256, 0, stream, in, out, words);
}
cudaError_t launch_narrow(const u64 *in, u32 *out, int64_t words, cudaStream_t stream) {
    if (words == 0) return cudaSuccess;
    return launch(narrow_kernel, (unsigned)((words + 1023) / 1024), 256, 0, stream, in, out, words);
}

}  // namespace hecuda
