// galois.cu -- Galois automorphisms f(x) -> f(x^g) on RNS polynomials (SURVEY.md 8f rank 1).
//
//   PolyRq<Coeff>.applyGalois   PolyRq/Galois.swift:115-141  (GaloisCoeffIterator :18-60)
//   PolyRq<Eval>.applyGalois    PolyRq/Galois.swift:151-166  (GaloisEvalIterator :62-98)
//
// Both are written as gathers so the stores are coalesced: the reference scatters out[(i g) mod N] = +-in[i]; the
// inverse map is i = (e g^-1 mod 2N) mod N with a sign flip when (e g^-1 mod 2N) >= N.
#include "kernels.cuh"

namespace hecuda {

__global__ void __launch_bounds__(256) galois_coeff_kernel(const u64 *__restrict__ in, int64_t in_poly_stride,
                                                          u64 *__restrict__ out, int64_t out_poly_stride,
                                                          const __grid_constant__ RowModuli c, int logn,
                                                          unsigned g_inv) {
    const int n = 1 << logn;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int row = blockIdx.y;
    const int64_t poly = blockIdx.z;
    const unsigned raw = ((unsigned)e * g_inv) & (2u * n - 1u);
    const unsigned src = raw & (n - 1u);
    const u64 v = in[poly * in_poly_stride + (int64_t)row * n + src];
    const u64 p = c.p[row];
    out[poly * out_poly_stride + (int64_t)row * n + e] = (raw >= (unsigned)n && v != 0) ? p - v : v;
}

__global__ void __launch_bounds__(256) galois_eval_kernel(const u64 *__restrict__ in, u64 *__restrict__ out, int rows,
                                                         int logn, unsigned g) {
    const int n = 1 << logn;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t base = ((int64_t)blockIdx.z * rows + blockIdx.y) * n;
    const unsigned reversed = __brev((unsigned)(i + n)) >> (31 - logn);          // bit-reverse over logn + 1 bits
    const unsigned raw = (unsigned)(((unsigned long long)g * reversed) >> 1) & (n - 1u);
    const unsigned src = logn ? (__brev(raw) >> (32 - logn)) : 0u;
    out[base + i] = in[base + src];
}

// PolyRq<Coeff>.multiplyPowerOfX (PolyRq.swift:398-422) as a gather: out[c] = +-in[(c - s) mod N], s = power mod 2N
__global__ void __launch_bounds__(256) monomial_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                      const __grid_constant__ RowModuli c, int logn, unsigned s) {
    const int n = 1 << logn;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int row = blockIdx.y;
    const int64_t base = ((int64_t)blockIdx.z * c.rows + row) * n;
    const unsigned raw = ((unsigned)e - s) & (2u * n - 1u);
    const u64 v = in[base + (raw & (n - 1u))];
    out[base + e] = (raw >= (unsigned)n && v != 0) ? c.p[row] - v : v;
}

cudaError_t launch_multiply_power_of_x(const Context &ctx, const NttRowMap &map, long long power, const u64 *in, u64 *out,
                                       int64_t polys, cudaStream_t stream) {
    if (polys == 0) return cudaSuccess;
    const RowModuli c = row_moduli(ctx, map);
    const long long two_n = 2 * ctx.n;
    long long s = power % two_n;
    if (s < 0) s += two_n;
    const int threads = coeff_threads(ctx.n);
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), (unsigned)c.rows, (unsigned)chunk);
        return launch(monomial_kernel, grid, threads, 0, stream, in + done * c.rows * ctx.n, out + done * c.rows * ctx.n, c,
                      ctx.logn, (unsigned)s);
    });
}

static unsigned inverse_mod_pow2(unsigned g, unsigned two_n) {  // g odd
    unsigned inv = g;
    for (int i = 0; i < 5; ++i) inv *= 2u - g * inv;
    return inv & (two_n - 1u);
}

cudaError_t launch_galois_coeff(const Context &ctx, const NttRowMap &map, unsigned element, const u64 *in,
                                int64_t in_poly_stride, u64 *out, int64_t out_poly_stride, int64_t polys,
                                cudaStream_t stream) {
    if (polys == 0) return cudaSuccess;
    const RowModuli c = row_moduli(ctx, map);
    const unsigned g_inv = inverse_mod_pow2(element, 2u * (unsigned)ctx.n);
    const int threads = coeff_threads(ctx.n);
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), (unsigned)c.rows, (unsigned)chunk);
        return launch(galois_coeff_kernel, grid, threads, 0, stream, in + done * in_poly_stride, in_poly_stride,
                      out + done * out_poly_stride, out_poly_stride, c, ctx.logn, g_inv);
    });
}

cudaError_t launch_galois_eval(const Context &ctx, int rows, unsigned element, const u64 *in, u64 *out, int64_t polys,
                               cudaStream_t stream) {
    if (polys == 0) return cudaSuccess;
    const int threads = coeff_threads(ctx.n);
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), (unsigned)rows, (unsigned)chunk);
        return launch(galois_eval_kernel, grid, threads, 0, stream, in + done * rows * ctx.n, out + done * rows * ctx.n, rows,
                      ctx.logn, element);
    });
}

}  // namespace hecuda
