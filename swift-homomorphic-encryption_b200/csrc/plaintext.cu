// plaintext.cu -- the plaintext side of Bfv on the device: SIMD encode / decode and ciphertext +- plaintext.
//
//   encodeSimd / decodeSimd          Encoding.swift:197-245     (generateEncodingMatrix, inverse / forward NTT mod t)
//   Bfv.encode(..., moduliCount:)    Bfv+Encode.swift:45-50     (+ Plaintext.convertToEvalFormat, Plaintext.swift:149-171)
//   Bfv.decodeEval                   Bfv+Encode.swift:76-80     (Plaintext.convertToCoeffFormat, Plaintext.swift:176-194)
//   plaintextTranslate               Bfv+Encrypt.swift:75-139   (addAssignCoeff / subAssignCoeff, Bfv.swift:110-117;
//                                                                 HeScheme.subCoeff = plaintext + -ciphertext, :1540-1542)
//
// The encode / decode pipelines are compositions of one gather kernel (writes coalesced) and the row NTT kernels on the
// plaintext modulus' slot (Context::slot_t); the translate is one coefficient-wise kernel.  All enqueue on one stream.
#include <cstdint>

#include "../../include/hecuda.h"
#include "kernels.cuh"
#include "ntt_fast.cuh"

namespace hecuda {

namespace {

constexpr int kThreads = 256;

template <int OP>
__device__ __forceinline__ u64 translate_one(u64 x, u64 v, u64 q) {
    if (OP == HECUDA_PLAINTEXT_ADD) return add_mod(x, v, q);
    if (OP == HECUDA_PLAINTEXT_SUB) return sub_mod(x, v, q);
    return sub_mod(v, x, q);  // SUB_FROM: -x + v
}

// A thread owns two adjacent coefficient columns of one ciphertext (blockIdx.y) over all l rows of every polynomial.
// VEC: 16-byte loads / stores (all pointers 16-byte aligned).  ct and out may be the same buffer: every element is read
// and written by the same thread.  rest: 0 = leave polys 1.. alone (in place), 1 = copy them, 2 = negate them.
template <int OP, bool VEC>
__global__ void __launch_bounds__(kThreads) plaintext_translate_kernel(const u64 *ct, u64 *out, const u64 *__restrict__ pt,
                                                                      long long pt_stride, int polys, int rest,
                                                                      const __grid_constant__ TranslateConsts c, int n) {
    const int col = 2 * (blockIdx.x * blockDim.x + threadIdx.x);
    if (col >= n) return;
    const long long item = blockIdx.y;
    const long long base = item * polys * c.l * (long long)n + col;
    const u64 *src = ct + base;
    u64 *dst = out + base;
    const u64 *p = pt + item * pt_stride + col;
    u64 m0, m1;
    if (VEC) {
        const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(p);
        m0 = v.x;
        m1 = v.y;
    } else {
        m0 = p[0];
        m1 = p[1];
    }
    const u64 adj0 = translate_adjust(m0, c), adj1 = translate_adjust(m1, c);
    for (int r = 0; r < c.l; ++r) {
        const u64 q = c.q[r], w = c.delta[r], wp = c.delta_p[r];
        const long long o = (long long)r * n;
        u64 x0, x1;
        if (VEC) {
            const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(src + o);
            x0 = v.x;
            x1 = v.y;
        } else {
            x0 = src[o];
            x1 = src[o + 1];
        }
        x0 = translate_one<OP>(x0, add_mod(shoup_mul(m0, w, wp, q), adj0, q), q);
        x1 = translate_one<OP>(x1, add_mod(shoup_mul(m1, w, wp, q), adj1, q), q);
        if (VEC) {
            *reinterpret_cast<ulonglong2 *>(dst + o) = make_ulonglong2(x0, x1);
        } else {
            dst[o] = x0;
            dst[o + 1] = x1;
        }
    }
    if (rest == 0) return;
    for (int k = 1; k < polys; ++k)
        for (int r = 0; r < c.l; ++r) {
            const long long o = ((long long)k * c.l + r) * n;
            const u64 q = c.q[r];
            u64 x0, x1;
            if (VEC) {
                const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(src + o);
                x0 = v.x;
                x1 = v.y;
            } else {
                x0 = src[o];
                x1 = src[o + 1];
            }
            if (rest == 2) {  // negateMod (Scalar.swift:167-175)
                x0 = x0 ? q - x0 : 0;
                x1 = x1 ? q - x1 : 0;
            }
            if (VEC) {
                *reinterpret_cast<ulonglong2 *>(dst + o) = make_ulonglong2(x0, x1);
            } else {
                dst[o] = x0;
                dst[o + 1] = x1;
            }
        }
}

// encodeSimd's scatter as a gather: Eval position j of plaintext `item` takes slot inverse[j] (0 past value_count)
__global__ void __launch_bounds__(kThreads) simd_encode_kernel(const u64 *__restrict__ values, int value_count,
                                                              const int32_t *__restrict__ inverse, u64 *__restrict__ out,
                                                              int n) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long item = blockIdx.y;
    const int slot = inverse[j];
    out[item * n + j] = slot < value_count ? values[item * value_count + slot] : 0;
}

// decodeSimd's gather: slot i of plaintext `item` is Eval position matrix[i]
__global__ void __launch_bounds__(kThreads) simd_decode_kernel(const u64 *__restrict__ eval, const int32_t *__restrict__ matrix,
                                                              u64 *__restrict__ values, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long item = blockIdx.y;
    values[item * n + i] = eval[item * n + matrix[i]];
}

// convertToCoeffFormat's un-centering of row 0 (Plaintext.swift:183-189): x >= tThreshold ? x - (q_0 - t) : x
__global__ void __launch_bounds__(kThreads) uncenter_kernel(u64 *data, u64 threshold, u64 increment, long long words) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    const u64 x = data[i];
    data[i] = x >= threshold ? x - increment : x;
}

}  // namespace

// at most kMaxGridYZ rows per call when N = 2^15 (the split path puts rows in grid z)
cudaError_t ntt_single(const Context &ctx, int slot, bool inverse, const u64 *in, u64 *out, int64_t rows, cudaStream_t s) {
    const NttRowMap map = ctx.map_single(slot);
    return for_each_part(rows, [&](int64_t done, int64_t part) {
        return inverse ? launch_ntt_inverse(ctx, map, in + done * ctx.n, out + done * ctx.n, part, kScalePlain, s)
                       : launch_ntt_forward(ctx, map, in + done * ctx.n, out + done * ctx.n, part, s);
    }, ctx.logn >= fast::kSplitLogN ? kMaxGridYZ : rows);
}

namespace {

cudaError_t launch_simd_gather(const Context &ctx, bool encode, const u64 *in, int value_count, u64 *out, int64_t count,
                               cudaStream_t s) {
    const int threads = coeff_threads(ctx.n);
    const unsigned gx = (unsigned)((ctx.n + threads - 1) / threads);
    return for_each_part(count, [&](int64_t done, int64_t part) {
        if (encode)
            return launch(simd_encode_kernel, dim3(gx, (unsigned)part), threads, 0, s, in + done * value_count, value_count,
                          ctx.d_simd_inverse, out + done * ctx.n, (int)ctx.n);
        return launch(simd_decode_kernel, dim3(gx, (unsigned)part), threads, 0, s, in + done * ctx.n, ctx.d_simd_matrix,
                      out + done * ctx.n, (int)ctx.n);
    });
}

}  // namespace

size_t simd_scratch_words(const Context &ctx, bool encode, int l) { return encode && l == 0 ? 0 : (size_t)ctx.n; }

cudaError_t launch_encode_simd(const Context &ctx, const u64 *values, int value_count, int l, u64 *out, u64 *scratch,
                               int64_t count, cudaStream_t s) {
    if (count == 0) return cudaSuccess;
    if (!ctx.simd || value_count < 0 || value_count > ctx.n || l < 0 || l > ctx.L) return cudaErrorInvalidValue;
    u64 *coeff = l == 0 ? out : scratch;
    cudaError_t e;
    if ((e = launch_simd_gather(ctx, true, values, value_count, coeff, count, s)) != cudaSuccess) return e;
    if ((e = ntt_single(ctx, ctx.slot_t(), true, coeff, coeff, count, s)) != cudaSuccess) return e;
    if (l == 0) return cudaSuccess;
    return launch_plaintext_to_eval(ctx, coeff, l, out, count, s);
}

cudaError_t launch_decode_simd(const Context &ctx, const u64 *plain, int l, u64 *values, u64 *scratch, int64_t count,
                               cudaStream_t s) {
    if (count == 0) return cudaSuccess;
    if (!ctx.simd || l < 0 || l > ctx.L) return cudaErrorInvalidValue;
    cudaError_t e;
    if (l == 0) {
        if ((e = ntt_single(ctx, ctx.slot_t(), false, plain, scratch, count, s)) != cudaSuccess) return e;
    } else {
        // row 0 of each Eval plaintext -> Coeff mod q_0 -> centered lift undone -> Eval mod t
        const size_t row_bytes = sizeof(u64) * (size_t)ctx.n;
        if ((e = cudaMemcpy2DAsync(scratch, row_bytes, plain, row_bytes * l, row_bytes, (size_t)count,
                                   cudaMemcpyDeviceToDevice, s)) != cudaSuccess)
            return e;
        if ((e = ntt_single(ctx, ctx.slot_q(0), true, scratch, scratch, count, s)) != cudaSuccess) return e;
        const long long words = (long long)count * ctx.n;
        if ((e = launch(uncenter_kernel, (unsigned)((words + kThreads - 1) / kThreads), kThreads, 0, s, scratch,
                        (ctx.t + 1) / 2, ctx.q[0] - ctx.t, words)) != cudaSuccess)
            return e;
        if ((e = ntt_single(ctx, ctx.slot_t(), false, scratch, scratch, count, s)) != cudaSuccess) return e;
    }
    return launch_simd_gather(ctx, false, scratch, 0, values, count, s);
}

cudaError_t launch_plaintext_translate(const Context &ctx, const u64 *ct, int polys, int l, const u64 *pt, bool broadcast,
                                       int op, u64 *out, int64_t batch, cudaStream_t s) {
    if (batch == 0) return cudaSuccess;
    if (l < 1 || l > ctx.L || polys < 1 || op < HECUDA_PLAINTEXT_ADD || op > HECUDA_PLAINTEXT_SUB_FROM)
        return cudaErrorInvalidValue;
    const TranslateConsts &c = ctx.translate[l];
    const int rest = op == HECUDA_PLAINTEXT_SUB_FROM ? 2 : (out != ct ? 1 : 0);
    const bool vec = (((uintptr_t)ct | (uintptr_t)out | (uintptr_t)pt) & 15) == 0;
    const int threads = coeff_threads(ctx.n / 2);
    const unsigned gx = (unsigned)((ctx.n / 2 + threads - 1) / threads);
    const long long pt_stride = broadcast ? 0 : ctx.n;
    const int64_t ct_words = (int64_t)polys * l * ctx.n;
    // [op][vec]
    static void (*const kernels[3][2])(const u64 *, u64 *, const u64 *, long long, int, int, TranslateConsts, int) = {
        {plaintext_translate_kernel<HECUDA_PLAINTEXT_ADD, false>, plaintext_translate_kernel<HECUDA_PLAINTEXT_ADD, true>},
        {plaintext_translate_kernel<HECUDA_PLAINTEXT_SUB, false>, plaintext_translate_kernel<HECUDA_PLAINTEXT_SUB, true>},
        {plaintext_translate_kernel<HECUDA_PLAINTEXT_SUB_FROM, false>, plaintext_translate_kernel<HECUDA_PLAINTEXT_SUB_FROM, true>}};
    return for_each_part(batch, [&](int64_t done, int64_t part) {
        return launch(kernels[op][vec], dim3(gx, (unsigned)part), threads, 0, s, ct + done * ct_words, out + done * ct_words,
                      pt + done * pt_stride, pt_stride, polys, rest, c, (int)ctx.n);
    });
}

}  // namespace hecuda
