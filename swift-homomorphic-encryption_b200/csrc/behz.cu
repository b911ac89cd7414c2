// behz.cu -- the coefficient-wise BEHZ steps of BFV ct x ct multiply (eprint 2016/510).
//
//   lift   = _RnsTool.liftQToQBsk            RnsTool.swift:324-368  (+ RnsBaseConverter.swift:97-143)
//   tensor = Bfv.multiplyWithoutScaling      Bfv+Multiply.swift:80-82
//   floor  = _RnsTool.floorQBskToQ           RnsTool.swift:378-456
//
// Layout/launch: lift and floor run persistent CTAs over column tiles (below); the tensor kernels give a thread two
// adjacent coefficient columns (16-byte loads/stores, coalesced along the coefficient axis; rows are strided by N) and
// select the polynomial with blockIdx.y/z, so there is no integer division.
// Arithmetic: each step evaluates the reference's chain of exact modular operations with pre-multiplied constants
// (context.hpp) as one 128-bit multiply-accumulate pass per output residue followed by ONE Montgomery reduction
// (the 2^64 factor lives in the constants); the stored residues are the same canonical values.  All kernels are
// instruction-issue bound (64-bit integer multiplies), not HBM bound -- see DESIGN.md.
#include "kernels.cuh"
#include "ntt_fast.cuh"

namespace hecuda {

constexpr int kThreads = 128;

template <int COLS>
struct Cols {
    u64 v[COLS];
};
template <int COLS>
__device__ __forceinline__ Cols<COLS> ldc(const u64 *p) {
    Cols<COLS> r;
    if (COLS % 2 == 0) {
#pragma unroll
        for (int h = 0; h < COLS / 2; ++h) {
            const ulonglong2 t = reinterpret_cast<const ulonglong2 *>(p)[h];
            r.v[2 * h] = t.x;
            r.v[2 * h + (COLS > 1)] = t.y;
        }
    } else {
        r.v[0] = *p;
    }
    return r;
}
template <int COLS>
__device__ __forceinline__ void stc(u64 *p, const u64 (&v)[COLS]) {
    if (COLS % 2 == 0) {
#pragma unroll
        for (int h = 0; h < COLS / 2; ++h)
            reinterpret_cast<ulonglong2 *>(p)[h] = make_ulonglong2(v[2 * h], v[2 * h + (COLS > 1)]);
    } else {
        *p = v[0];
    }
}

// ---- lift and floor: CTA b owns column tile b, kThreads * COLS consecutive coefficients of one polynomial (1-D grid,
// tiles of a polynomial adjacent).  A thread issues every row load of its tile before any arithmetic, so it makes one
// trip to memory, and the many resident CTAs overlap one another's loads and multiplies.  Two columns per thread
// (16-byte accesses) up to L = 8; one above that, which keeps every instantiation free of spills.
template <int L>
struct BehzCols {
    static constexpr int value = L <= 8 ? 2 : 1;
};

struct ColTiles {
    long long count;  // polynomials << shift
    int shift;        // log2(tiles per polynomial); N < kThreads * COLS: one partial tile per polynomial
};

// first column of tile t owned by this thread
template <int COLS>
__device__ __forceinline__ int tile_col(long long t, const ColTiles &tl) {
    return (int)(t & ((1ll << tl.shift) - 1)) * (kThreads * COLS) + (int)threadIdx.x * COLS;
}

template <int ROWS, int COLS>
__device__ __forceinline__ void load_rows(Cols<COLS> (&x)[ROWS], const u64 *src, int64_t n) {
#pragma unroll
    for (int i = 0; i < ROWS; ++i) x[i] = ldc<COLS>(src + (int64_t)i * n);
}

// Bounds (checked for the actual moduli by Context::create): every 128-bit accumulator below stays < 2^127 and the
// Montgomery-reduced sums are < 2p (lift, f_j, out_i: one or two conditional subtractions) or < 4p (alpha).
// H: every b_j is h 2^32 + 1 (LiftConsts / FloorConsts::h_primes), so the reductions modulo b_j take mont_reduce_h.
// Output polynomial g = (item * ops + op) * 2^pin_shift + pin of ext (ops = 2 with rhs, else 1) is the lift of input
// polynomial item * 2^pin_shift + pin of lhs (op 0) or rhs (op 1); it has the L + 1 auxiliary rows, after the L Q rows
// when Q_ROWS.
template <int L, bool H, bool Q_ROWS>
__global__ void __launch_bounds__(kThreads) lift_kernel(const u64 *__restrict__ lhs, const u64 *__restrict__ rhs,
                                                       int pin_shift, u64 *__restrict__ ext,
                                                       const __grid_constant__ LiftConsts c, int n, ColTiles tiles) {
    constexpr int COLS = BehzCols<L>::value, ROWS_OUT = Q_ROWS ? 2 * L + 1 : L + 1, AUX0 = Q_ROWS ? L : 0;
    if ((int)threadIdx.x * COLS >= n) return;
    const int op_shift = rhs ? 1 : 0;
    auto src_of = [&](long long t) {
        const int64_t g = t >> tiles.shift, item = g >> (pin_shift + op_shift);
        const int64_t pin = g & ((1 << pin_shift) - 1);
        const u64 *base = (op_shift && ((g >> pin_shift) & 1)) ? rhs : lhs;
        return base + ((item << pin_shift) + pin) * L * n + tile_col<COLS>(t, tiles);
    };
    const long long t = blockIdx.x;
    {
        Cols<COLS> x[L];
        load_rows<L, COLS>(x, src_of(t), n);
        u64 *dst = ext + (t >> tiles.shift) * ROWS_OUT * n + tile_col<COLS>(t, tiles);
        u64 z[COLS][L];
        u32 acc_mt[COLS];
#pragma unroll
        for (int k = 0; k < COLS; ++k) acc_mt[k] = 0;
#pragma unroll
        for (int i = 0; i < L; ++i) {
            if (Q_ROWS) stc<COLS>(dst + (int64_t)i * n, x[i].v);
#pragma unroll
            for (int k = 0; k < COLS; ++k) {
                // canonical: z is reinterpreted mod b_j and mod m~ below
                z[k][i] = shoup_mul(x[i].v[k], c.in_w[i], c.in_wp[i], c.q[i]);
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
            stc<COLS>(dst + (int64_t)(AUX0 + j) * n, o);
        }
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

// Q_SCALED: the Q rows arrive as y_i = [x_i (Q/q_i)^-1]_{q_i} already (the inverse NTT's kScaleTMontFloor)
// (a minimum of one CTA per SM from L = 8 lets ptxas use the registers that keep those instantiations free of spills)
template <int L, bool H, bool Q_SCALED>
__global__ void __launch_bounds__(kThreads, L >= 8 ? 1 : 0) floor_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                        const __grid_constant__ FloorConsts c, int n, ColTiles tiles) {
    constexpr int R = 2 * L + 1, COLS = BehzCols<L>::value;
    if ((int)threadIdx.x * COLS >= n) return;
    const long long t = blockIdx.x;
    {
        Cols<COLS> x[R];
        load_rows<R, COLS>(x, in + (t >> tiles.shift) * R * n + tile_col<COLS>(t, tiles), n);
        u64 y[COLS][L];
#pragma unroll
        for (int i = 0; i < L; ++i)
#pragma unroll
            for (int k = 0; k < COLS; ++k)
                y[k][i] = Q_SCALED ? x[i].v[k] : shoup_mul(x[i].v[k], c.inq_w[i], c.inq_wp[i], c.q[i]);
        // approximateFloor, RnsTool.swift:378-398: f_j = (x_bj - FBC(x_Q)_j) Q^-1 mod b_j; for j < L the constants
        // carry (B/b_j)^-1 as well, so f_j is w_j of the conversion below (canonical); f_L is kept lazy (< 2 m_sk)
        u64 f[COLS][L + 1];
#pragma unroll
        for (int j = 0; j <= L; ++j) {
#pragma unroll
            for (int k = 0; k < COLS; ++k) {
                u128 acc = (u128)x[L + j].v[k] * c.fq[j];
#pragma unroll
                for (int i = 0; i < L; ++i) mac128(acc, y[k][i], c.fmat[j][i]);
                const u64 red = mont_reduce_c<H>(acc, c.b[j], c.b_ninv[j]);
                f[k][j] = j == L ? red : c.wide_sums ? barrett64(red, c.b[j], c.b_mu1[j]) : csub(red, c.b[j]);
            }
        }
        // convertApproximateBskToQ, RnsTool.swift:402-450
        const u64 msk = c.b[L];
        u64 outv[L][COLS];
#pragma unroll
        for (int k = 0; k < COLS; ++k) {
            const u64 *w = f[k];  // w_i = [f_i (B/b_i)^-1]_{b_i}, canonical: reinterpreted mod m_sk and q_i
            u128 acc = (u128)f[k][L] * c.a_msk;
#pragma unroll
            for (int i = 0; i < L; ++i) mac128(acc, w[i], c.amat[i]);
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
        u64 *dst = out + (t >> tiles.shift) * L * n + tile_col<COLS>(t, tiles);
#pragma unroll
        for (int i = 0; i < L; ++i) stc<COLS>(dst + (int64_t)i * n, outv[i]);
    }
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
    u64 y[kMaxL], f[kMaxL + 1];
    for (int i = 0; i < L; ++i) y[i] = shoup_mul(src[(int64_t)i * n], c.inq_w[i], c.inq_wp[i], c.q[i]);
    for (int j = 0; j <= L; ++j) {  // f_j for j < L is w_j (FloorConsts)
        u128 acc = (u128)src[(int64_t)(L + j) * n] * c.fq[j];
        for (int i = 0; i < L; ++i) mac128(acc, y[i], c.fmat[j][i]);
        const u64 red = mont_reduce(acc, c.b[j], c.b_ninv[j]);
        f[j] = j == L ? red : barrett64(red, c.b[j], c.b_mu1[j]);
    }
    const u64 *w = f;
    const u64 msk = c.b[L];
    u128 acc = (u128)f[L] * c.a_msk;
    for (int i = 0; i < L; ++i) mac128(acc, w[i], c.amat[i]);
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

static ColTiles col_tiles(int64_t n, int64_t polys, int cols) {
    ColTiles tl;
    tl.shift = 0;
    while (((int64_t)kThreads * cols << tl.shift) < n) ++tl.shift;
    tl.count = (long long)polys << tl.shift;
    return tl;
}

template <bool H, bool Q_ROWS>
static cudaError_t launch_lift_tiles(const Context &ctx, const u64 *lhs, const u64 *rhs, int pin_shift, u64 *ext,
                                     int64_t polys_out, const LiftConsts &consts, cudaStream_t stream) {
    cudaError_t e;
    ColTiles tl;
    HE_DISPATCH_L(ctx.L, (tl = col_tiles(ctx.n, polys_out, BehzCols<LL>::value),
                          e = tl.count > 0x7fffffffLL ? cudaErrorInvalidConfiguration  // one CTA per tile: gridDim.x
                                                    : launch(lift_kernel<LL, H, Q_ROWS>, (unsigned)tl.count, kThreads, 0,
                                                             stream, lhs, rhs, pin_shift, ext, consts, (int)ctx.n, tl)));
    return e;
}
template <bool H, bool Q_SCALED>
static cudaError_t launch_floor_tiles(const Context &ctx, const u64 *in, u64 *out, int64_t polys,
                                      const FloorConsts &consts, cudaStream_t stream) {
    cudaError_t e;
    ColTiles tl;
    HE_DISPATCH_L(ctx.L, (tl = col_tiles(ctx.n, polys, BehzCols<LL>::value),
                          e = tl.count > 0x7fffffffLL ? cudaErrorInvalidConfiguration  // one CTA per tile: gridDim.x
                                                    : launch(floor_kernel<LL, H, Q_SCALED>, (unsigned)tl.count, kThreads, 0,
                                                             stream, in, out, consts, (int)ctx.n, tl)));
    return e;
}

// grid over (coefficients, polys) with polys folded into y (<= 32768) and z: the kernels above 16 moduli
static inline dim3 poly_grid(int64_t n, int64_t polys) {
    const unsigned gx = (unsigned)((n + kThreads - 1) / kThreads);
    const int64_t gy = polys < 32768 ? polys : 32768;
    return dim3(gx ? gx : 1, (unsigned)gy, (unsigned)((polys + gy - 1) / gy));
}

static cudaError_t launch_lift_generic(const Context &ctx, const u64 *in, int polys_in, u64 *ext, int ext_polys,
                                       int out_poly_offset, int64_t items, cudaStream_t stream, const LiftConsts &consts,
                                       bool q_rows) {
    int64_t polys = items * polys_in;
    const int64_t pstride_in = (int64_t)ctx.L * ctx.n;
    // the z dimension must divide exactly: launch in slabs of y = 32768 polys, then the remainder
    while (polys > 0) {
        int64_t slab = polys >= 32768 ? (polys / 32768) * 32768 : polys;
        const cudaError_t e = launch(lift_generic_kernel, poly_grid(ctx.n, slab), kThreads, 0, stream, in, polys_in, ext,
                                     ext_polys, out_poly_offset, consts, (int)ctx.n, q_rows);
        if (e != cudaSuccess) return e;
        // advance whole items only (32768 is even and polys_in is 1 or 2)
        in += slab * pstride_in;
        ext += (slab / polys_in) * (int64_t)ext_polys * (q_rows ? 2 * ctx.L + 1 : ctx.L + 1) * ctx.n;
        polys -= slab;
    }
    return cudaSuccess;
}

cudaError_t launch_lift(const Context &ctx, const u64 *lhs, const u64 *rhs, int polys_in, u64 *ext, int64_t items,
                        cudaStream_t stream, bool reference_base, bool q_rows) {
    const LiftConsts &consts = reference_base ? ctx.lift : ctx.lift_mul;
    if (items == 0) return cudaSuccess;
    if (polys_in != 1 && polys_in != 2) return cudaErrorInvalidValue;
    const int ops = rhs ? 2 : 1;
    if (ctx.L > 16) {
        cudaError_t e = launch_lift_generic(ctx, lhs, polys_in, ext, ops * polys_in, 0, items, stream, consts, q_rows);
        if (e == cudaSuccess && rhs)
            e = launch_lift_generic(ctx, rhs, polys_in, ext, ops * polys_in, polys_in, items, stream, consts, q_rows);
        return e;
    }
    const int64_t polys_out = items * ops * polys_in;
    const int pin_shift = polys_in == 2 ? 1 : 0;
    auto lift_tiles = consts.h_primes ? (q_rows ? launch_lift_tiles<true, true> : launch_lift_tiles<true, false>)
                                      : (q_rows ? launch_lift_tiles<false, true> : launch_lift_tiles<false, false>);
    return lift_tiles(ctx, lhs, rhs, pin_shift, ext, polys_out, consts, stream);
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
    bool any_h = false;
    for (int r = 0; r < tc.R; ++r) any_h |= tc.h[r] != 0;
    auto k = any_h ? tensor_kernel<2, true> : tensor_kernel<2, false>;  // N >= 2: two columns per thread
    const unsigned gx = (unsigned)((ctx.n / 2 + kThreads - 1) / kThreads);
    return for_each_part(items, [&](int64_t done, int64_t chunk) {
        dim3 grid(gx ? gx : 1, (unsigned)tc.R, (unsigned)chunk);
        return launch(k, grid, kThreads, 0, stream, ext + done * 4 * tc.R * ctx.n, ten + done * 3 * tc.R * ctx.n, tc, (int)ctx.n);
    });
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
    return for_each_part(groups, [&](int64_t done, int64_t chunk) {
        dim3 grid(gx ? gx : 1, (unsigned)tc.R, (unsigned)chunk);
        return launch(tensor_sum_kernel, grid, kThreads, 0, stream, ext + done * pairs * 4 * tc.R * ctx.n,
                      ten + done * 3 * tc.R * ctx.n, tc, (int)ctx.n, pairs);
    });
}

bool floor_takes_scaled_q(const Context &ctx) { return ctx.L <= 16; }

cudaError_t launch_floor(const Context &ctx, const u64 *in, u64 *out, int64_t polys, cudaStream_t stream,
                         bool reference_base, bool q_scaled) {
    if (polys == 0) return cudaSuccess;
    const FloorConsts &consts = reference_base ? ctx.floor : ctx.floor_mul;
    if (ctx.L <= 16) {
        auto floor_tiles = consts.h_primes ? (q_scaled ? launch_floor_tiles<true, true> : launch_floor_tiles<true, false>)
                                           : (q_scaled ? launch_floor_tiles<false, true> : launch_floor_tiles<false, false>);
        return floor_tiles(ctx, in, out, polys, consts, stream);
    }
    if (q_scaled) return cudaErrorInvalidValue;  // floor_takes_scaled_q
    const int R = 2 * ctx.L + 1;
    while (polys > 0) {
        int64_t slab = polys >= 32768 ? (polys / 32768) * 32768 : polys;
        const cudaError_t e = launch(floor_generic_kernel, poly_grid(ctx.n, slab), kThreads, 0, stream, in, out, consts, (int)ctx.n);
        if (e != cudaSuccess) return e;
        in += slab * (int64_t)R * ctx.n;
        out += slab * (int64_t)ctx.L * ctx.n;
        polys -= slab;
    }
    return cudaSuccess;
}

}  // namespace hecuda
