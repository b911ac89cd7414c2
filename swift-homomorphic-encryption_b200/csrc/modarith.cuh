// modarith.cuh -- 64-bit modular arithmetic primitives for sm_90a (and host, for the SIMT emulation tests).
//
// Device-side equivalents of the reference's scalar layer (Sources/ModularArithmetic/Modulus.swift,
// Scalar.swift).  What must match the reference is the *value* stored back into a polynomial -- always the
// canonical residue in [0, p) (PolyRq.swift:36,85-95) -- not how it is reduced, so the lazy ranges below are
// chosen for the GPU's instruction mix (IMAD-bound), not copied from the CPU code.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define HE_HD __host__ __device__ __forceinline__
#define HE_D __device__ __forceinline__
#else
#define HE_HD inline
#define HE_D inline
#endif

namespace hecuda {

typedef unsigned long long u64;
typedef unsigned int u32;

HE_HD u64 mulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

// x >= p ? x - p : x        (reference: subtractIfExceeds, Scalar.swift:160-166)
HE_HD u64 csub(u64 x, u64 p) { return x >= p ? x - p : x; }
HE_HD u64 add_mod(u64 a, u64 b, u64 p) { return csub(a + b, p); }
HE_HD u64 sub_mod(u64 a, u64 b, u64 p) { return csub(a + p - b, p); }

// Shoup constant multiply, lazy: returns x*w mod p in [0, 2p) for ANY x < 2^64, p < 2^63.
// wp = floor(w * 2^64 / p).   (reference: MultiplyConstantModulus.multiplyModLazy, Modulus.swift:401-410)
HE_HD u64 shoup_lazy(u64 x, u64 w, u64 wp, u64 p) {
    u64 q = mulhi64(x, wp);
    return x * w - q * p;
}
HE_HD u64 shoup_mul(u64 x, u64 w, u64 wp, u64 p) { return csub(shoup_lazy(x, w, wp, p), p); }

// Single-word Barrett: x mod p for any x < 2^64; mu1 = floor(2^64 / p).  (Modulus.swift:258-263)
HE_HD u64 barrett64(u64 x, u64 p, u64 mu1) {
    u64 q = mulhi64(x, mu1);
    return csub(x - q * p, p);
}

// 128-bit value as two words.
struct u128w {
    u64 lo, hi;
};
HE_HD u128w mul_wide(u64 a, u64 b) {
    u128w r;
    r.lo = a * b;
    r.hi = mulhi64(a, b);
    return r;
}
HE_HD void mac_wide(u128w &acc, u64 a, u64 b) {
    u64 lo = a * b;
    u64 hi = mulhi64(a, b);
    acc.lo += lo;
    acc.hi += hi + (acc.lo < lo ? 1ull : 0ull);
}

// Double-word Barrett: (hi:lo) mod p for any 128-bit value, p < 2^63; (mu_hi:mu_lo) = floor(2^128 / p).
// Only the low word of the quotient estimate is needed because the result is < 2p < 2^64.
// (reference: ReduceModulus.reduce(_: DoubleWidth), Modulus.swift:319-325)
HE_HD u64 barrett128(u128w x, u64 p, u64 mu_hi, u64 mu_lo) {
    // qhat = floor(x * mu / 2^128), low 64 bits
    u64 ll_hi = mulhi64(x.lo, mu_lo);
    u64 lh_lo = x.lo * mu_hi, lh_hi = mulhi64(x.lo, mu_hi);
    u64 hl_lo = x.hi * mu_lo, hl_hi = mulhi64(x.hi, mu_lo);
    u64 hh_lo = x.hi * mu_hi;
    u64 mid = ll_hi + lh_lo;
    u64 c1 = mid < ll_hi ? 1ull : 0ull;
    u64 mid2 = mid + hl_lo;
    u64 c2 = mid2 < mid ? 1ull : 0ull;
    u64 q = hh_lo + lh_hi + hl_hi + c1 + c2;
    return csub(x.lo - q * p, p);
}

// ---- 128-bit accumulation + Montgomery reduction (the workhorse of the base-conversion kernels).
// acc = sum of 64x64 products; mont_reduce returns acc * 2^-64 mod p in [0, (acc >> 64) + p), with
// ninv = -p^-1 mod 2^64.  The 2^64 factor is folded into precomputed constants (or into the scaling of the
// following inverse NTT), so results are the same canonical residues as the reference's Barrett path
// (RnsBaseConverter.swift:117-143 accumulates in DoubleWidth and reduces once, like this).
typedef unsigned __int128 u128;
HE_HD void mac128(u128 &acc, u64 a, u64 b) { acc += (u128)a * b; }
HE_HD u64 mont_reduce(u128 acc, u64 p, u64 ninv) {
    const u64 lo = (u64)acc, hi = (u64)(acc >> 64);
    const u64 m = lo * ninv;
    return hi + mulhi64(m, p) + (lo != 0 ? 1ull : 0ull);
}
// mont_reduce for p = h 2^32 + 1 < 2^55 (the multiply's 55-bit auxiliary primes, context.cu), the same value in every
// case.  ninv = h 2^32 - 1, so m = lo ninv mod 2^64 = ((lo0 h) << 32) - lo takes one 32-bit multiply, and with
// m p = m0 + 2^32 (m1 + m0 h) + 2^64 m1 h, hi64(m p) = m1 h + hi32(m0 h + m1) takes two 32 x 32 -> 64 ones.  The generic
// form spends three multiplies on m and four wide ones on the 64-bit mulhi.
HE_HD u64 mont_reduce_h(u128 acc, u64 p) {
    const u64 lo = (u64)acc, hi = (u64)(acc >> 64);
    const u32 h = (u32)(p >> 32), lo0 = (u32)lo, lo1 = (u32)(lo >> 32);
    const u32 m0 = 0u - lo0, m1 = lo0 * h - lo1 - (lo0 != 0 ? 1u : 0u);  // m = 2^32 m1 + m0
    return hi + (u64)m1 * h + (((u64)m0 * h + m1) >> 32) + (lo != 0 ? 1ull : 0ull);
}
template <bool H>
HE_HD u64 mont_reduce_c(u128 acc, u64 p, u64 ninv) { return H ? mont_reduce_h(acc, p) : mont_reduce(acc, p, ninv); }

// Product Barrett: (hi:lo) mod p for values < 4 p^2, p < 2^61 (tensor products and sums of two of them).
// s = bits(p) - 2, mu = floor(2^(s+64) / p).  Result canonical.
// (reference: ReduceModulus.reduceProduct, Modulus.swift:349-360, which covers x < p^2 with one csub;
//  the extra conditional subtractions here extend the admissible range.)
HE_HD u64 barrett_prod(u128w x, u64 p, u64 mu, int s) {
    u64 xs = (x.lo >> s) | (x.hi << (64 - s));
    u64 q = mulhi64(xs, mu);
    u64 r = x.lo - q * p;
    r = csub(r, 4 * p);
    r = csub(r, 2 * p);
    return csub(r, p);
}

}  // namespace hecuda
