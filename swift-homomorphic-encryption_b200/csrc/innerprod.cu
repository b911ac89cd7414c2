// innerprod.cu -- lazy ciphertext x plaintext inner products and plaintext Eval conversion (SURVEY.md 8f rank 2).
//
//   Bfv.innerProduct(ciphertexts:plaintexts:)   Bfv/Bfv.swift:476-505  (lazyMultiply :388-400, reduce :365-394)
//   PolyRq.addingLazyProduct                    PolyRq/PolyRq.swift:210-225
//   Plaintext.convertToEvalFormat               Plaintext.swift:149-171
//
// out[o][p][r][c] = sum_k cts[k][p][r][c] * pts[o][k][r][c] mod q_r over the present plaintexts -- the MulPir
// first-dimension scan (IndexPir/PirUtil.swift:437-442): `out_count` database rows against the same `terms` query
// ciphertexts.  The plaintexts are streamed from HBM exactly once (ld.global.cs); the ciphertexts are re-read through
// L2.  128-bit lazy accumulation like the reference, one double-word Barrett at the end (and every max_terms terms).
#include "kernels.cuh"

namespace hecuda {

struct IpConsts {
    int l;
    long long max_terms;  // maxLazyProductAccumulationCount (PolyContext.swift:246-253)
    u64 p[kMaxL], mu_hi[kMaxL], mu_lo[kMaxL];
};

__device__ __forceinline__ u128w to_w(u128 v) {
    u128w r;
    r.lo = (u64)v;
    r.hi = (u64)(v >> 64);
    return r;
}

// One output row (blockIdx.z) per thread: more rows per thread, each reusing the query-ciphertext values fetched
// through L2, cost registers and measured slower.
template <int NPOLY, bool HAS_PRESENT>
__global__ void __launch_bounds__(128) inner_product_plain_kernel(const u64 *__restrict__ cts, const u64 *__restrict__ pts,
                                                                 const unsigned char *__restrict__ present,
                                                                 u64 *__restrict__ out,
                                                                 const __grid_constant__ IpConsts c, int n,
                                                                 long long terms) {
    const int coeff = (blockIdx.x * 128 + threadIdx.x) * 2;
    if (coeff >= n) return;
    const int r = blockIdx.y, l = c.l;
    const long long o = blockIdx.z;
    const u64 p = c.p[r], mu_hi = c.mu_hi[r], mu_lo = c.mu_lo[r];
    u128 acc[NPOLY][2];
#pragma unroll
    for (int q = 0; q < NPOLY; ++q) acc[q][0] = acc[q][1] = 0;
    const long long pt_stride = (long long)l * n, ct_stride = (long long)NPOLY * l * n;
    const u64 *ct = cts + (long long)r * n + coeff;
    const u64 *pt = pts + ((o * terms) * l + r) * (long long)n + coeff;
    const unsigned char *pres = HAS_PRESENT ? present + o * terms : nullptr;
    long long since_reduce = 0;
#pragma unroll 2
    for (long long k = 0; k < terms; ++k) {
        ulonglong2 cv[NPOLY];
#pragma unroll
        for (int q = 0; q < NPOLY; ++q)
            cv[q] = __ldg(reinterpret_cast<const ulonglong2 *>(ct + k * ct_stride + (long long)q * pt_stride));
        if (!HAS_PRESENT || pres[k]) {  // nil plaintext (Bfv.swift:493), uniform across the block
            const ulonglong2 pv = __ldcs(reinterpret_cast<const ulonglong2 *>(pt + k * pt_stride));
#pragma unroll
            for (int q = 0; q < NPOLY; ++q) {
                mac128(acc[q][0], cv[q].x, pv.x);
                mac128(acc[q][1], cv[q].y, pv.y);
            }
        }
        if (++since_reduce >= c.max_terms) {  // reduceInPlace, Bfv.swift:365-377
            since_reduce = 0;
#pragma unroll
            for (int q = 0; q < NPOLY; ++q) {
                acc[q][0] = barrett128(to_w(acc[q][0]), p, mu_hi, mu_lo);
                acc[q][1] = barrett128(to_w(acc[q][1]), p, mu_hi, mu_lo);
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NPOLY; ++q) {  // reduceToCiphertext, Bfv.swift:380-394
        u64 *dst = out + (((o * NPOLY + q) * l + r) * (long long)n) + coeff;
        *reinterpret_cast<ulonglong2 *>(dst) =
            make_ulonglong2(barrett128(to_w(acc[q][0]), p, mu_hi, mu_lo), barrett128(to_w(acc[q][1]), p, mu_hi, mu_lo));
    }
}

cudaError_t launch_inner_product_plain(const Context &ctx, const u64 *cts, int npoly, int l, int64_t terms, const u64 *pts,
                                       const unsigned char *present, u64 *out, int64_t out_count, cudaStream_t stream) {
    if (out_count == 0) return cudaSuccess;
    if (npoly < 1 || npoly > 3 || l < 1 || l > ctx.L || ctx.n < 2) return cudaErrorInvalidValue;
    IpConsts c;
    c.l = l;
    u64 qmax = 0;
    for (int r = 0; r < l; ++r) {
        const ModSlot &S = ctx.slots[ctx.slot_q(r)].dev;
        c.p[r] = S.p;
        c.mu_hi[r] = S.mu_hi;
        c.mu_lo[r] = S.mu_lo;
        qmax = S.p > qmax ? S.p : qmax;
    }
    const u128 max_product = (u128)(qmax - 1) * (qmax - 1);
    const u128 max_count = ((~(u128)0) - qmax) / max_product;
    c.max_terms = max_count > (u128)0x7fffffffffffffffLL ? 0x7fffffffffffffffLL : (long long)max_count;
    const unsigned gx = (unsigned)((ctx.n / 2 + 127) / 128);
    // [npoly - 1][present given]
    static void (*const kernels[3][2])(const u64 *, const u64 *, const unsigned char *, u64 *, IpConsts, int, long long) = {
        {inner_product_plain_kernel<1, false>, inner_product_plain_kernel<1, true>},
        {inner_product_plain_kernel<2, false>, inner_product_plain_kernel<2, true>},
        {inner_product_plain_kernel<3, false>, inner_product_plain_kernel<3, true>}};
    for (int64_t done = 0; done < out_count;) {
        const int64_t chunk = (out_count - done) > 65535 ? 65535 : (out_count - done);
        dim3 grid(gx ? gx : 1, (unsigned)l, (unsigned)chunk);
        const u64 *pt = pts + done * terms * l * ctx.n;
        const unsigned char *pr = present ? present + done * terms : nullptr;
        u64 *o = out + done * npoly * l * ctx.n;
        ++g_kernel_launches;
        kernels[npoly - 1][pr != nullptr]<<<grid, 128, 0, stream>>>(cts, pt, pr, o, c, (int)ctx.n, terms);
        done += chunk;
    }
    return cudaGetLastError();
}

// ---- the same scan for moduli below 2^31 (the reference's default PIR parameters, 27 / 28 / 28 bits): the database
// rows are kept as uint32 (half the bytes to stream), a product of two residues fits 62 bits, so one IMAD.WIDE with a
// 64-bit accumulator replaces the 128-bit multiply-accumulate, reduced (single-word Barrett) every max_terms terms.
struct IpSmallConsts {
    int l;
    int max_terms;
    u64 p[kMaxL], mu1[kMaxL];
};
// One database row (blockIdx.z) per thread: at the config-4 shape (437 terms x 75 rows) so few rows make the grid, not
// L2, the limit.
template <int NPOLY, bool HAS_PRESENT>
__global__ void __launch_bounds__(128) inner_product_plain_small_kernel(const u64 *__restrict__ cts, const u32 *__restrict__ pts,
                                                                       const unsigned char *__restrict__ present,
                                                                       u64 *__restrict__ out,
                                                                       const __grid_constant__ IpSmallConsts c, int n,
                                                                       long long terms) {
    const int coeff = (blockIdx.x * 128 + threadIdx.x) * 4;  // four adjacent coefficients: 16-byte loads of the uint32 rows
    if (coeff >= n) return;
    const int r = blockIdx.y, l = c.l;
    const long long o = blockIdx.z;
    const u64 p = c.p[r], mu1 = c.mu1[r];
    u64 acc[NPOLY][4];
#pragma unroll
    for (int q = 0; q < NPOLY; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0;
    const long long pt_stride = (long long)l * n, ct_stride = (long long)NPOLY * l * n;
    const u64 *ct = cts + (long long)r * n + coeff;
    const u32 *pt = pts + ((o * terms) * l + r) * (long long)n + coeff;
    const unsigned char *pres = HAS_PRESENT ? present + o * terms : nullptr;
    int since_reduce = 0;
#pragma unroll 2
    for (long long k = 0; k < terms; ++k) {
        const uint4 pv = __ldcs(reinterpret_cast<const uint4 *>(pt + k * pt_stride));
#pragma unroll
        for (int q = 0; q < NPOLY; ++q) {
            const u64 *cq = ct + k * ct_stride + (long long)q * pt_stride;
            const ulonglong2 c01 = __ldg(reinterpret_cast<const ulonglong2 *>(cq));
            const ulonglong2 c23 = __ldg(reinterpret_cast<const ulonglong2 *>(cq + 2));
            if (HAS_PRESENT && !pres[k]) continue;  // nil plaintext (Bfv.swift:493), uniform across the block
            acc[q][0] += (u64)(u32)c01.x * pv.x;
            acc[q][1] += (u64)(u32)c01.y * pv.y;
            acc[q][2] += (u64)(u32)c23.x * pv.z;
            acc[q][3] += (u64)(u32)c23.y * pv.w;
        }
        if (++since_reduce >= c.max_terms) {  // reduceInPlace, Bfv.swift:365-377
            since_reduce = 0;
#pragma unroll
            for (int q = 0; q < NPOLY; ++q)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[q][j] = barrett64(acc[q][j], p, mu1);
        }
    }
#pragma unroll
    for (int q = 0; q < NPOLY; ++q) {  // reduceToCiphertext, Bfv.swift:380-394
        u64 *dst = out + (((o * NPOLY + q) * l + r) * (long long)n) + coeff;
        reinterpret_cast<ulonglong2 *>(dst)[0] = make_ulonglong2(barrett64(acc[q][0], p, mu1), barrett64(acc[q][1], p, mu1));
        reinterpret_cast<ulonglong2 *>(dst)[1] = make_ulonglong2(barrett64(acc[q][2], p, mu1), barrett64(acc[q][3], p, mu1));
    }
}

bool inner_product_plain_small_supported(const Context &ctx, int l) {
    if (ctx.n < 4) return false;
    for (int r = 0; r < l; ++r)
        if (ctx.slots[ctx.slot_q(r)].dev.bits > 31) return false;
    return true;
}

cudaError_t launch_inner_product_plain_small(const Context &ctx, const u64 *cts, int npoly, int l, int64_t terms, const u32 *pts,
                                             const unsigned char *present, u64 *out, int64_t out_count, cudaStream_t stream) {
    if (out_count == 0) return cudaSuccess;
    if (npoly < 1 || npoly > 3 || l < 1 || l > ctx.L || !inner_product_plain_small_supported(ctx, l)) return cudaErrorInvalidValue;
    IpSmallConsts c;
    c.l = l;
    u64 qmax = 0;
    for (int r = 0; r < l; ++r) {
        const ModSlot &S = ctx.slots[ctx.slot_q(r)].dev;
        c.p[r] = S.p;
        c.mu1[r] = S.mu1;
        qmax = S.p > qmax ? S.p : qmax;
    }
    // a reduced accumulator (< p) plus max_terms products (< (p-1)^2 each) must stay below 2^64
    const u128 room = (~(u128)0 >> 64) - qmax;
    const u128 max_count = room / ((u128)(qmax - 1) * (qmax - 1));
    c.max_terms = max_count > 0x7fffffff ? 0x7fffffff : (int)max_count;
    if (c.max_terms < 1) return cudaErrorInvalidValue;
    const unsigned gx = (unsigned)((ctx.n / 4 + 127) / 128);
    // [npoly - 1][present given]
    static void (*const kernels[3][2])(const u64 *, const u32 *, const unsigned char *, u64 *, IpSmallConsts, int, long long) = {
        {inner_product_plain_small_kernel<1, false>, inner_product_plain_small_kernel<1, true>},
        {inner_product_plain_small_kernel<2, false>, inner_product_plain_small_kernel<2, true>},
        {inner_product_plain_small_kernel<3, false>, inner_product_plain_small_kernel<3, true>}};
    for (int64_t done = 0; done < out_count;) {
        const int64_t chunk = (out_count - done) > 65535 ? 65535 : (out_count - done);
        dim3 grid(gx ? gx : 1, (unsigned)l, (unsigned)chunk);
        const u32 *pt = pts + done * terms * l * ctx.n;
        const unsigned char *pr = present ? present + done * terms : nullptr;
        u64 *o = out + done * npoly * l * ctx.n;
        ++g_kernel_launches;
        kernels[npoly - 1][pr != nullptr]<<<grid, 128, 0, stream>>>(cts, pt, pr, o, c, (int)ctx.n, terms);
        done += chunk;
    }
    return cudaGetLastError();
}

// Plaintext.convertToEvalFormat, Plaintext.swift:149-171: centered lift mod each q_r (the forward NTT follows)
__global__ void __launch_bounds__(256) plaintext_lift_kernel(const u64 *__restrict__ plain, u64 *__restrict__ out,
                                                            const __grid_constant__ IpConsts c, u64 t, int n) {
    const int coeff = blockIdx.x * blockDim.x + threadIdx.x;
    if (coeff >= n) return;
    const int r = blockIdx.y;
    const long long item = blockIdx.z;
    const u64 v = plain[item * n + coeff];
    const u64 threshold = (t + 1) >> 1;  // RnsTool.tThreshold, RnsTool.swift:123-125
    out[(item * c.l + r) * n + coeff] = v < threshold ? v : v + (c.p[r] - t);  // tIncrement, RnsTool.swift:168
}

cudaError_t launch_plaintext_to_eval(const Context &ctx, const u64 *plain, int l, u64 *out, int64_t count,
                                     cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    if (l < 1 || l > ctx.L) return cudaErrorInvalidValue;
    IpConsts c;
    c.l = l;
    c.max_terms = 0;
    for (int r = 0; r < l; ++r) c.p[r] = ctx.slots[ctx.slot_q(r)].dev.p;
    const int threads = ctx.n >= 256 ? 256 : (ctx.n < 32 ? 32 : (int)ctx.n);
    for (int64_t done = 0; done < count;) {
        const int64_t chunk = (count - done) > 65535 ? 65535 : (count - done);
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), (unsigned)l, (unsigned)chunk);
        ++g_kernel_launches;
        plaintext_lift_kernel<<<grid, threads, 0, stream>>>(plain + done * ctx.n, out + done * l * ctx.n, c, ctx.t, (int)ctx.n);
        done += chunk;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return launch_ntt_forward(ctx, ctx.map_q(l), out, out, count * l, stream);
}

}  // namespace hecuda
