// behz.cu -- the coefficient-wise BEHZ steps of BFV ct x ct multiply (eprint 2016/510).
//
//   lift   = _RnsTool.liftQToQBsk            RnsTool.swift:324-368  (+ RnsBaseConverter.swift:97-143)
//   tensor = Bfv.multiplyWithoutScaling      Bfv+Multiply.swift:80-82
//   floor  = _RnsTool.floorQBskToQ           RnsTool.swift:378-456
//
// Layout/launch: a thread owns two adjacent coefficient columns (16-byte loads/stores, coalesced along the
// coefficient axis; rows are strided by N); blockIdx.y/z select the polynomial, so there is no integer division.
// Arithmetic: each step evaluates the reference's chain of exact modular operations with pre-multiplied constants
// (context.hpp) as one 128-bit multiply-accumulate pass per output residue followed by ONE Montgomery reduction
// (the 2^64 factor lives in the constants); the stored residues are the same canonical values.  All kernels are
// instruction-issue bound (64-bit integer multiplies), not HBM bound -- see DESIGN.md.
#include <cstdlib>

#include "kernels.cuh"
#include "ntt_fast.cuh"

namespace hecuda {

constexpr int kThreads = 128;

// columns per thread: 2 (16-byte accesses) by default; HECUDA_BEHZ_COLS=1 selects 1 (more warps, 8-byte accesses)
static int cols_per_thread() {
    static const int v = [] {
        const char *e = std::getenv("HECUDA_BEHZ_COLS");
        return (e && e[0] == '1') ? 1 : 2;
    }();
    return v;
}

template <int COLS>
struct Cols {
    u64 v[COLS];
};
template <int COLS>
__device__ __forceinline__ Cols<COLS> ldc(const u64 *p) {
    Cols<COLS> r;
    if (COLS == 2) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2 *>(p);
        r.v[0] = t.x;
        r.v[COLS - 1] = t.y;
    } else {
        r.v[0] = *p;
    }
    return r;
}
template <int COLS>
__device__ __forceinline__ void stc(u64 *p, const u64 (&v)[COLS]) {
    if (COLS == 2) *reinterpret_cast<ulonglong2 *>(p) = make_ulonglong2(v[0], v[COLS - 1]);
    else *p = v[0];
}

// Bounds (checked for the actual moduli by Context::create): every 128-bit accumulator below stays < 2^127 and the
// Montgomery-reduced sums are < 2p (lift, f_j, out_i: one or two conditional subtractions) or < 4p (alpha).
// H: every b_j is h 2^32 + 1 (LiftConsts / FloorConsts::h_primes), so the reductions modulo b_j take mont_reduce_h.
template <int L, int COLS, bool H>
__global__ void __launch_bounds__(kThreads) lift_kernel(const u64 *__restrict__ in, int polys_in, u64 *__restrict__ ext,
                                                       int ext_polys, int out_poly_offset,
                                                       const __grid_constant__ LiftConsts c, int n, bool q_rows) {
    const int rows_out = q_rows ? 2 * L + 1 : L + 1, aux0 = q_rows ? L : 0;
    const int coeff = (blockIdx.x * kThreads + threadIdx.x) * COLS;
    if (coeff >= n) return;
    const int64_t poly = (int64_t)blockIdx.z * gridDim.y + blockIdx.y;  // index among items * polys_in
    const int64_t item = polys_in == 2 ? (poly >> 1) : poly / polys_in;  // (no 64-bit division on the hot path)
    const int pin = (int)(poly - item * polys_in);
    const u64 *src = in + poly * L * n + coeff;
    u64 *dst = ext + ((item * ext_polys + out_poly_offset + pin) * rows_out) * n + coeff;
    u64 z[COLS][L];
    u32 acc_mt[COLS];
#pragma unroll
    for (int k = 0; k < COLS; ++k) acc_mt[k] = 0;
#pragma unroll
    for (int i = 0; i < L; ++i) {
        const Cols<COLS> x = ldc<COLS>(src + (int64_t)i * n);
        if (q_rows) stc<COLS>(dst + (int64_t)i * n, x.v);
#pragma unroll
        for (int k = 0; k < COLS; ++k) {
            // canonical: z is reinterpreted mod b_j and mod m~ below
            z[k][i] = shoup_mul(x.v[k], c.in_w[i], c.in_wp[i], c.q[i]);
            acc_mt[k] += (u32)z[k][i] * c.punct_mt[i];
        }
    }
    u32 r[COLS];
    bool neg[COLS];
#pragma unroll
    for (int k = 0; k < COLS; ++k) {
        r[k] = (acc_mt[k] * c.neg_inv_q_mt) & c.mt_mask;  // [-x' Q^-1]_{m~}, RnsTool.swift:343-348
        neg[k] = r[k] >= c.mt_half;                       // centered representative r - m~ (:357-360)
    }
#pragma unroll
    for (int j = 0; j <= L; ++j) {
        u64 o[COLS];
#pragma unroll
        for (int k = 0; k < COLS; ++k) {
            const u64 rc = neg[k] ? (u64)r[k] + c.neg_off[j] : (u64)r[k];
            u128 acc = (u128)rc * c.qr[j];
#pragma unroll
            for (int i = 0; i < L; ++i) mac128(acc, z[k][i], c.mat[j][i]);
            const u64 red = mont_reduce_c<H>(acc, c.b[j], c.b_ninv[j]);
            o[k] = c.wide_sums ? barrett64(red, c.b[j], c.b_mu1[j]) : csub(red, c.b[j]);
        }
        stc<COLS>(dst + (int64_t)(aux0 + j) * n, o);
    }
}

// Tensor product in Montgomery form: out = a b 2^-64 mod p (canonical).  The missing 2^64 is restored by the
// kScaleTMont scaling of the inverse NTT that always follows (Bfv+Multiply.swift:80-82 then :40-41).
struct TensorConsts {
    int R;
    u64 p[kMaxRows], ninv[kMaxRows];
    unsigned char h[kMaxRows];  // p = h 2^32 + 1 < 2^55: mont_reduce_h
};

template <int COLS, bool H>
__device__ __forceinline__ void tensor_cols(const Cols<COLS> &a0, const Cols<COLS> &a1, const Cols<COLS> &b0,
                                            const Cols<COLS> &b1, u64 p, u64 ninv, u64 (&o0)[COLS], u64 (&o1)[COLS],
                                            u64 (&o2)[COLS]) {
#pragma unroll
    for (int k = 0; k < COLS; ++k) {
        o0[k] = csub(mont_reduce_c<H>((u128)a0.v[k] * b0.v[k], p, ninv), p);
        u128 m = (u128)a0.v[k] * b1.v[k];
        mac128(m, a1.v[k], b0.v[k]);
        o1[k] = csub(mont_reduce_c<H>(m, p, ninv), p);
        o2[k] = csub(mont_reduce_c<H>((u128)a1.v[k] * b1.v[k], p, ninv), p);
    }
}

// ANY_H: some row's prime is h 2^32 + 1 (the others keep the kernel without that branch)
template <int COLS, bool ANY_H>
__global__ void __launch_bounds__(kThreads) tensor_kernel(const u64 *__restrict__ ext, u64 *__restrict__ ten,
                                                         const __grid_constant__ TensorConsts c, int n) {
    const int R = c.R;
    const int row = blockIdx.y;
    const int64_t item = blockIdx.z;
    const int coeff = (blockIdx.x * kThreads + threadIdx.x) * COLS;
    if (coeff >= n) return;
    const u64 p = c.p[row], ninv = c.ninv[row];
    const u64 *e = ext + (item * 4 * R + row) * n + coeff;
    const int64_t ps = (int64_t)R * n;
    const Cols<COLS> a0 = ldc<COLS>(e), a1 = ldc<COLS>(e + ps), b0 = ldc<COLS>(e + 2 * ps), b1 = ldc<COLS>(e + 3 * ps);
    u64 *o = ten + (item * 3 * R + row) * n + coeff;
    u64 o0[COLS], o1[COLS], o2[COLS];
    if (ANY_H && c.h[row]) tensor_cols<COLS, true>(a0, a1, b0, b1, p, ninv, o0, o1, o2);
    else tensor_cols<COLS, false>(a0, a1, b0, b1, p, ninv, o0, o1, o2);
    stc<COLS>(o, o0);
    stc<COLS>(o + ps, o1);
    stc<COLS>(o + 2 * ps, o2);
}

// Sum of tensor products over `pairs` ciphertext pairs (Bfv.innerProduct(_:_:), Bfv.swift:315-361: lazyMultiply
// accumulates l0 r0, l0 r1 + l1 r0, l1 r1 in DoubleWidth, reduceToCiphertext reduces once).  ext[group][pair][4][R][N]
// (Eval) -> ten[group][3][R][N] in Montgomery form like tensor_kernel.  max_pairs bounds the lazy accumulation
// (maxLazyProductAccumulationCount / 2, Bfv.swift:331); beyond it the accumulators are Barrett-reduced in place.
struct TensorSumConsts {
    int R;
    long long max_pairs;
    u64 p[kMaxRows], ninv[kMaxRows], mu1[kMaxRows], mu_hi[kMaxRows], mu_lo[kMaxRows];
};

__global__ void __launch_bounds__(kThreads) tensor_sum_kernel(const u64 *__restrict__ ext, u64 *__restrict__ ten,
                                                             const __grid_constant__ TensorSumConsts c, int n,
                                                             long long pairs) {
    const int R = c.R;
    const int row = blockIdx.y;
    const int64_t group = blockIdx.z;
    const int coeff = (blockIdx.x * kThreads + threadIdx.x) * 2;
    if (coeff >= n) return;
    const u64 p = c.p[row], ninv = c.ninv[row];
    const int64_t ps = (int64_t)R * n;
    const u64 *e = ext + (group * pairs * 4 * R + row) * n + coeff;
    u128 a0[2] = {0, 0}, a1[2] = {0, 0}, a2[2] = {0, 0};
    long long since = 0;
    for (long long k = 0; k < pairs; ++k, e += 4 * ps) {
        const Cols<2> l0 = ldc<2>(e), l1 = ldc<2>(e + ps), r0 = ldc<2>(e + 2 * ps), r1 = ldc<2>(e + 3 * ps);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            mac128(a0[j], l0.v[j], r0.v[j]);
            mac128(a1[j], l0.v[j], r1.v[j]);
            mac128(a1[j], l1.v[j], r0.v[j]);
            mac128(a2[j], l1.v[j], r1.v[j]);
        }
        if (++since >= c.max_pairs) {  // reduceInPlace, Bfv.swift:365-377
            since = 0;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                u128w w0 = {(u64)a0[j], (u64)(a0[j] >> 64)}, w1 = {(u64)a1[j], (u64)(a1[j] >> 64)},
                      w2 = {(u64)a2[j], (u64)(a2[j] >> 64)};
                a0[j] = barrett128(w0, p, c.mu_hi[row], c.mu_lo[row]);
                a1[j] = barrett128(w1, p, c.mu_hi[row], c.mu_lo[row]);
                a2[j] = barrett128(w2, p, c.mu_hi[row], c.mu_lo[row]);
            }
        }
    }
    u64 *o = ten + (group * 3 * R + row) * n + coeff;
    u64 o0[2], o1[2], o2[2];
    const u64 mu1 = c.mu1[row];
#pragma unroll
    for (int j = 0; j < 2; ++j) {  // sums < 2^127 (max_pairs) -> Montgomery result < 2^63 + p; one single-word Barrett
        o0[j] = barrett64(mont_reduce(a0[j], p, ninv), p, mu1);
        o1[j] = barrett64(mont_reduce(a1[j], p, ninv), p, mu1);
        o2[j] = barrett64(mont_reduce(a2[j], p, ninv), p, mu1);
    }
    stc<2>(o, o0);
    stc<2>(o + ps, o1);
    stc<2>(o + 2 * ps, o2);
}

template <int L, int COLS, bool H>
__global__ void __launch_bounds__(kThreads) floor_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                        const __grid_constant__ FloorConsts c, int n) {
    constexpr int R = 2 * L + 1;
    const int coeff = (blockIdx.x * kThreads + threadIdx.x) * COLS;
    if (coeff >= n) return;
    const int64_t poly = (int64_t)blockIdx.z * gridDim.y + blockIdx.y;
    const u64 *src = in + poly * R * n + coeff;
    u64 *dst = out + poly * L * n + coeff;
    u64 y[COLS][L];
#pragma unroll
    for (int i = 0; i < L; ++i) {
        const Cols<COLS> x = ldc<COLS>(src + (int64_t)i * n);
#pragma unroll
        for (int k = 0; k < COLS; ++k) y[k][i] = shoup_mul(x.v[k], c.inq_w[i], c.inq_wp[i], c.q[i]);
    }
    // approximateFloor, RnsTool.swift:378-398: f_j = (x_bj - FBC(x_Q)_j) Q^-1 mod b_j   (kept lazy, < 2 b_j)
    u64 f[COLS][L + 1];
#pragma unroll
    for (int j = 0; j <= L; ++j) {
        const Cols<COLS> xb = ldc<COLS>(src + (int64_t)(L + j) * n);
#pragma unroll
        for (int k = 0; k < COLS; ++k) {
            u128 acc = (u128)xb.v[k] * c.fq[j];
#pragma unroll
            for (int i = 0; i < L; ++i) mac128(acc, y[k][i], c.fmat[j][i]);
            f[k][j] = mont_reduce_c<H>(acc, c.b[j], c.b_ninv[j]);
        }
    }
    // convertApproximateBskToQ, RnsTool.swift:402-450
    const u64 msk = c.b[L];
    u64 outv[L][COLS];
#pragma unroll
    for (int k = 0; k < COLS; ++k) {
        u64 w[L];
        u128 acc = (u128)f[k][L] * c.a_msk;
#pragma unroll
        for (int i = 0; i < L; ++i) {
            w[i] = shoup_mul(f[k][i], c.inb_w[i], c.inb_wp[i], c.b[i]);  // canonical: reinterpreted mod m_sk and q_i
            mac128(acc, w[i], c.amat[i]);
        }
        u64 alpha = mont_reduce_c<H>(acc, msk, c.b_ninv[L]);
        alpha = c.wide_sums ? barrett64(alpha, msk, c.msk_mu1) : csub(csub(csub(alpha, 4 * msk), 2 * msk), msk);
        const bool exceeds = alpha > (msk >> 1);
        const u64 alpha_c = exceeds ? msk - alpha : alpha;
#pragma unroll
        for (int i = 0; i < L; ++i) {
            u128 o = (u128)alpha_c * (exceeds ? c.b_mod_q[i] : c.neg_b_mod_q[i]);
#pragma unroll
            for (int kk = 0; kk < L; ++kk) mac128(o, w[kk], c.omat[i][kk]);
            outv[i][k] = csub(csub(mont_reduce(o, c.q[i], c.q_ninv[i]), 2 * c.q[i]), c.q[i]);
        }
    }
#pragma unroll
    for (int i = 0; i < L; ++i) stc<COLS>(dst + (int64_t)i * n, outv[i]);
}

// ---- more than 16 ciphertext moduli (the reference allows 32 coefficient moduli, EncryptionParameters.swift:148): the
// same arithmetic with run-time loop bounds, one column per thread, the per-modulus temporaries in local memory.  Such
// parameter sets are rare and slow on every platform; this keeps them correct rather than fast.
__global__ void __launch_bounds__(kThreads) lift_generic_kernel(const u64 *__restrict__ in, int polys_in, u64 *__restrict__ ext,
                                                               int ext_polys, int out_poly_offset,
                                                               const __grid_constant__ LiftConsts c, int n, bool q_rows) {
    const int L = c.L, rows_out = q_rows ? 2 * L + 1 : L + 1, aux0 = q_rows ? L : 0;
    const int coeff = blockIdx.x * kThreads + threadIdx.x;
    if (coeff >= n) return;
    const int64_t poly = (int64_t)blockIdx.z * gridDim.y + blockIdx.y;
    const int64_t item = poly / polys_in;
    const int pin = (int)(poly - item * polys_in);
    const u64 *src = in + poly * L * n + coeff;
    u64 *dst = ext + ((item * ext_polys + out_poly_offset + pin) * rows_out) * n + coeff;
    u64 z[kMaxL];
    u32 acc_mt = 0;
    for (int i = 0; i < L; ++i) {
        const u64 x = src[(int64_t)i * n];
        if (q_rows) dst[(int64_t)i * n] = x;
        z[i] = shoup_mul(x, c.in_w[i], c.in_wp[i], c.q[i]);
        acc_mt += (u32)z[i] * c.punct_mt[i];
    }
    const u32 r = (acc_mt * c.neg_inv_q_mt) & c.mt_mask;
    const bool neg = r >= c.mt_half;
    for (int j = 0; j <= L; ++j) {
        const u64 rc = neg ? (u64)r + c.neg_off[j] : (u64)r;
        u128 acc = (u128)rc * c.qr[j];
        for (int i = 0; i < L; ++i) mac128(acc, z[i], c.mat[j][i]);
        const u64 red = mont_reduce(acc, c.b[j], c.b_ninv[j]);
        dst[(int64_t)(aux0 + j) * n] = c.wide_sums ? barrett64(red, c.b[j], c.b_mu1[j]) : csub(red, c.b[j]);
    }
}

__global__ void __launch_bounds__(kThreads) floor_generic_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                                const __grid_constant__ FloorConsts c, int n) {
    const int L = c.L, R = 2 * L + 1;
    const int coeff = blockIdx.x * kThreads + threadIdx.x;
    if (coeff >= n) return;
    const int64_t poly = (int64_t)blockIdx.z * gridDim.y + blockIdx.y;
    const u64 *src = in + poly * R * n + coeff;
    u64 *dst = out + poly * L * n + coeff;
    u64 y[kMaxL], f[kMaxL + 1], w[kMaxL];
    for (int i = 0; i < L; ++i) y[i] = shoup_mul(src[(int64_t)i * n], c.inq_w[i], c.inq_wp[i], c.q[i]);
    for (int j = 0; j <= L; ++j) {
        u128 acc = (u128)src[(int64_t)(L + j) * n] * c.fq[j];
        for (int i = 0; i < L; ++i) mac128(acc, y[i], c.fmat[j][i]);
        f[j] = mont_reduce(acc, c.b[j], c.b_ninv[j]);
    }
    const u64 msk = c.b[L];
    u128 acc = (u128)f[L] * c.a_msk;
    for (int i = 0; i < L; ++i) {
        w[i] = shoup_mul(f[i], c.inb_w[i], c.inb_wp[i], c.b[i]);
        mac128(acc, w[i], c.amat[i]);
    }
    u64 alpha = mont_reduce(acc, msk, c.b_ninv[L]);
    alpha = c.wide_sums ? barrett64(alpha, msk, c.msk_mu1) : csub(csub(csub(alpha, 4 * msk), 2 * msk), msk);
    const bool exceeds = alpha > (msk >> 1);
    const u64 alpha_c = exceeds ? msk - alpha : alpha;
    for (int i = 0; i < L; ++i) {
        u128 o = (u128)alpha_c * (exceeds ? c.b_mod_q[i] : c.neg_b_mod_q[i]);
        for (int kk = 0; kk < L; ++kk) mac128(o, w[kk], c.omat[i][kk]);
        // (L + 1) b q / 2^64 may exceed 3q with this many moduli: finish with a Barrett reduction
        dst[(int64_t)i * n] = barrett64(mont_reduce(o, c.q[i], c.q_ninv[i]), c.q[i], c.q_mu1[i]);
    }
}

#define HE_DISPATCH_L(L_, CALL)                                                                                       \
    switch (L_) {                                                                                                     \
        case 1: { constexpr int LL = 1; CALL; } break;                                                                \
        case 2: { constexpr int LL = 2; CALL; } break;                                                                \
        case 3: { constexpr int LL = 3; CALL; } break;                                                                \
        case 4: { constexpr int LL = 4; CALL; } break;                                                                \
        case 5: { constexpr int LL = 5; CALL; } break;                                                                \
        case 6: { constexpr int LL = 6; CALL; } break;                                                                \
        case 7: { constexpr int LL = 7; CALL; } break;                                                                \
        case 8: { constexpr int LL = 8; CALL; } break;                                                                \
        case 9: { constexpr int LL = 9; CALL; } break;                                                                \
        case 10: { constexpr int LL = 10; CALL; } break;                                                              \
        case 11: { constexpr int LL = 11; CALL; } break;                                                              \
        case 12: { constexpr int LL = 12; CALL; } break;                                                              \
        case 13: { constexpr int LL = 13; CALL; } break;                                                              \
        case 14: { constexpr int LL = 14; CALL; } break;                                                              \
        case 15: { constexpr int LL = 15; CALL; } break;                                                              \
        case 16: { constexpr int LL = 16; CALL; } break;                                                              \
        default: return cudaErrorInvalidValue;                                                                        \
    }

template <int COLS, bool H>
static cudaError_t launch_lift_kernel(int L, dim3 grid, cudaStream_t stream, const u64 *in, int polys_in, u64 *ext,
                                      int ext_polys, int out_poly_offset, const LiftConsts &consts, int n, bool q_rows) {
    HE_DISPATCH_L(L, (lift_kernel<LL, COLS, H><<<grid, kThreads, 0, stream>>>(in, polys_in, ext, ext_polys, out_poly_offset,
                                                                              consts, n, q_rows)));
    return cudaSuccess;
}
template <int COLS, bool H>
static cudaError_t launch_floor_kernel(int L, dim3 grid, cudaStream_t stream, const u64 *in, u64 *out,
                                       const FloorConsts &consts, int n) {
    HE_DISPATCH_L(L, (floor_kernel<LL, COLS, H><<<grid, kThreads, 0, stream>>>(in, out, consts, n)));
    return cudaSuccess;
}

// grid over (coefficient pairs, polys) with polys folded into y (<= 32768) and z
static inline dim3 poly_grid(int64_t n, int64_t polys, int cols) {
    const unsigned gx = (unsigned)((n / cols + kThreads - 1) / kThreads);
    const int64_t gy = polys < 32768 ? polys : 32768;
    return dim3(gx ? gx : 1, (unsigned)gy, (unsigned)((polys + gy - 1) / gy));
}

cudaError_t launch_lift(const Context &ctx, const u64 *in, int polys_in, u64 *ext, int ext_polys, int out_poly_offset,
                        int64_t items, cudaStream_t stream, bool reference_base, bool q_rows) {
    const LiftConsts &consts = reference_base ? ctx.lift : ctx.lift_mul;
    int64_t polys = items * polys_in;
    if (polys == 0) return cudaSuccess;
    const int64_t pstride_in = (int64_t)ctx.L * ctx.n;
    // the z dimension must divide exactly: launch in slabs of y = 32768 polys, then the remainder
    while (polys > 0) {
        int64_t slab = polys >= 32768 ? (polys / 32768) * 32768 : polys;
        const int cols = ctx.L > 16 ? 1 : (ctx.n >= 2 ? cols_per_thread() : 1);
        const dim3 grid = poly_grid(ctx.n, slab, cols);
        ++g_kernel_launches;
        if (ctx.L > 16) {
            lift_generic_kernel<<<grid, kThreads, 0, stream>>>(in, polys_in, ext, ext_polys, out_poly_offset, consts, (int)ctx.n, q_rows);
        } else {
            auto launch = cols == 2 ? (consts.h_primes ? launch_lift_kernel<2, true> : launch_lift_kernel<2, false>)
                                    : (consts.h_primes ? launch_lift_kernel<1, true> : launch_lift_kernel<1, false>);
            const cudaError_t e = launch(ctx.L, grid, stream, in, polys_in, ext, ext_polys, out_poly_offset, consts, (int)ctx.n, q_rows);
            if (e != cudaSuccess) return e;
        }
        // advance whole items only (32768 is even and polys_in is 1 or 2)
        in += slab * pstride_in;
        ext += (slab / polys_in) * (int64_t)ext_polys * (q_rows ? 2 * ctx.L + 1 : ctx.L + 1) * ctx.n;
        polys -= slab;
    }
    return cudaGetLastError();
}

cudaError_t launch_tensor(const Context &ctx, const u64 *ext, u64 *ten, int64_t items, cudaStream_t stream,
                          bool reference_base) {
    if (items == 0) return cudaSuccess;
    TensorConsts tc;
    tc.R = 2 * ctx.L + 1;
    const NttRowMap map = reference_base ? ctx.map_qbsk() : ctx.map_qaux();
    for (int r = 0; r < tc.R; ++r) {
        tc.p[r] = ctx.slots[map.slot[r]].dev.p;
        tc.ninv[r] = ctx.slots[map.slot[r]].dev.ninv;
        tc.h[r] = fast::class_of_modulus(tc.p[r], ctx.slots[map.slot[r]].dev.bits) == fast::kNarrowH ? 1 : 0;
    }
    const int cols = ctx.n >= 2 ? cols_per_thread() : 1;
    bool any_h = false;
    for (int r = 0; r < tc.R; ++r) any_h |= tc.h[r] != 0;
    auto k = cols == 2 ? (any_h ? tensor_kernel<2, true> : tensor_kernel<2, false>) : (any_h ? tensor_kernel<1, true> : tensor_kernel<1, false>);
    const unsigned gx = (unsigned)((ctx.n / cols + kThreads - 1) / kThreads);
    for (int64_t done = 0; done < items;) {  // gridDim.z <= 65535
        const int64_t chunk = (items - done) > 65535 ? 65535 : (items - done);
        dim3 grid(gx ? gx : 1, (unsigned)tc.R, (unsigned)chunk);
        ++g_kernel_launches;
        k<<<grid, kThreads, 0, stream>>>(ext + done * 4 * tc.R * ctx.n, ten + done * 3 * tc.R * ctx.n, tc, (int)ctx.n);
        done += chunk;
    }
    return cudaGetLastError();
}

cudaError_t launch_tensor_sum(const Context &ctx, const u64 *ext, u64 *ten, int64_t pairs, int64_t groups,
                              cudaStream_t stream, bool reference_base) {
    if (groups == 0) return cudaSuccess;
    if (ctx.n < 2 || pairs < 1) return cudaErrorInvalidValue;
    TensorSumConsts tc;
    tc.R = 2 * ctx.L + 1;
    const NttRowMap map = reference_base ? ctx.map_qbsk() : ctx.map_qaux();
    u64 pmax = 0;
    for (int r = 0; r < tc.R; ++r) {
        const ModSlot &S = ctx.slots[map.slot[r]].dev;
        tc.p[r] = S.p;
        tc.ninv[r] = S.ninv;
        tc.mu1[r] = S.mu1;
        tc.mu_hi[r] = S.mu_hi;
        tc.mu_lo[r] = S.mu_lo;
        pmax = S.p > pmax ? S.p : pmax;
    }
    // each pair adds < 2 p^2 to the middle accumulator; keep every accumulator below 2^127
    const u128 per_pair = 2 * (u128)pmax * pmax;
    const u128 cap = (((u128)1) << 127) / per_pair;
    tc.max_pairs = cap < 1 ? 1 : (cap > (u128)0x7fffffffLL ? 0x7fffffffLL : (long long)cap);
    const unsigned gx = (unsigned)((ctx.n / 2 + kThreads - 1) / kThreads);
    for (int64_t done = 0; done < groups;) {
        const int64_t chunk = (groups - done) > 65535 ? 65535 : (groups - done);
        dim3 grid(gx ? gx : 1, (unsigned)tc.R, (unsigned)chunk);
        ++g_kernel_launches;
        tensor_sum_kernel<<<grid, kThreads, 0, stream>>>(ext + done * pairs * 4 * tc.R * ctx.n, ten + done * 3 * tc.R * ctx.n,
                                                         tc, (int)ctx.n, pairs);
        done += chunk;
    }
    return cudaGetLastError();
}

cudaError_t launch_floor(const Context &ctx, const u64 *in, u64 *out, int64_t polys, cudaStream_t stream,
                         bool reference_base) {
    if (polys == 0) return cudaSuccess;
    const FloorConsts &consts = reference_base ? ctx.floor : ctx.floor_mul;
    const int R = 2 * ctx.L + 1;
    while (polys > 0) {
        int64_t slab = polys >= 32768 ? (polys / 32768) * 32768 : polys;
        const int cols = ctx.L > 16 ? 1 : (ctx.n >= 2 ? cols_per_thread() : 1);
        const dim3 grid = poly_grid(ctx.n, slab, cols);
        ++g_kernel_launches;
        if (ctx.L > 16) {
            floor_generic_kernel<<<grid, kThreads, 0, stream>>>(in, out, consts, (int)ctx.n);
        } else {
            auto launch = cols == 2 ? (consts.h_primes ? launch_floor_kernel<2, true> : launch_floor_kernel<2, false>)
                                    : (consts.h_primes ? launch_floor_kernel<1, true> : launch_floor_kernel<1, false>);
            const cudaError_t e = launch(ctx.L, grid, stream, in, out, consts, (int)ctx.n);
            if (e != cudaSuccess) return e;
        }
        in += slab * (int64_t)R * ctx.n;
        out += slab * (int64_t)ctx.L * ctx.n;
        polys -= slab;
    }
    return cudaGetLastError();
}

}  // namespace hecuda
