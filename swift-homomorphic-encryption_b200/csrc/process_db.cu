// process_db.cu -- the server's own data into plaintexts on the device: MulPirServer.process's packing and
// PlaintextMatrix(signedValues:)'s .diagonal packing with its SIMD encoding.  The index arithmetic is in
// process_db.cuh; these kernels only apply it.  Both enqueue on one stream.
#include "kernels.cuh"

namespace hecuda {

namespace {

constexpr int kThreads = 256;

// One CTA per plaintext: every thread extracts its coefficients straight from the entry bytes; a block-wide OR says
// whether the plaintext is non-nil (MulPir.swift:480, 536: an all-zero plaintext is nil).
__global__ void __launch_bounds__(kThreads) pir_pack_kernel(const procdb::PirShape s, int n, long long first,
                                                           u64 *__restrict__ out, unsigned char *__restrict__ present) {
    const long long item = blockIdx.x;
    const procdb::PirPiece p = procdb::pir_piece(s, first + item);
    u64 *row = out + item * n;
    int any = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const u64 v = procdb::pir_coefficient(s, p, i);
        row[i] = v;
        any |= v != 0;
    }
    any = __syncthreads_or(any);
    if (threadIdx.x == 0) present[item] = any ? 1 : 0;
}

// Eval position j of plaintext `first + blockIdx.y` takes SIMD slot inverse[j] of its diagonal chunk: the signed
// conversion, the diagonal gather, the half-row rotation and the encodeSimd scatter in one pass.  resident: plaintexts
// are counted in hecuda_pnns_matrix's slot order instead of diagonalPlaintexts' order.  A value outside the centered
// range sets *bad.
__global__ void __launch_bounds__(kThreads) pnns_gather_kernel(const long long *__restrict__ values,
                                                              const procdb::PnnsShape s, u64 t, int reduce, int resident,
                                                              const int32_t *__restrict__ inverse, long long first,
                                                              u64 *__restrict__ out, int *bad) {
    const int n = 1 << s.logn;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long item = first + blockIdx.y;
    int d;
    long long r;
    bool live = true;
    if (resident)
        live = procdb::pnns_resident(s, item, d, r);
    else
        procdb::pnns_plaintext(s, item, d, r);
    u64 v = 0;
    if (live) {
        const long long at = procdb::pnns_element(s, d, r, inverse[j]);
        if (at >= 0) {
            bool wrong = false;
            v = procdb::pnns_signed_value(values[at], t, reduce != 0, wrong);
            if (wrong) *bad = 1;
        }
    }
    out[(long long)blockIdx.y * n + j] = v;
}

}  // namespace

cudaError_t launch_pir_pack(const procdb::PirShape &s, int n, int64_t first, int64_t items, u64 *out,
                            unsigned char *present, cudaStream_t stream) {
    if (items == 0) return cudaSuccess;
    return launch(pir_pack_kernel, (unsigned)items, coeff_threads(n), 0, stream, s, n, (long long)first, out, present);
}

cudaError_t launch_pnns_diagonal(const Context &ctx, const procdb::PnnsShape &s, const int64_t *values, bool reduce,
                                 bool resident, int64_t first, int64_t items, u64 *out, int *bad, cudaStream_t stream) {
    if (items == 0) return cudaSuccess;
    if (!ctx.simd) return cudaErrorInvalidValue;
    const int threads = coeff_threads(ctx.n);
    const unsigned gx = (unsigned)((ctx.n + threads - 1) / threads);
    const cudaError_t e = for_each_part(items, [&](int64_t done, int64_t part) {
        return launch(pnns_gather_kernel, dim3(gx, (unsigned)part), threads, 0, stream, (const long long *)values, s, ctx.t,
                      reduce ? 1 : 0, resident ? 1 : 0, ctx.d_simd_inverse, (long long)(first + done), out + done * ctx.n, bad);
    });
    if (e != cudaSuccess) return e;
    // encodeSimd's inverse NTT mod t (Encoding.swift:206-214)
    return ntt_single(ctx, ctx.slot_t(), true, out, out, items, stream);
}

}  // namespace hecuda
