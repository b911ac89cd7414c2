// hostmath.hpp -- setup-time number theory for the device context (host only).
//
// Produces exactly the constants the reference precomputes (SURVEY.md section 8 row a15):
//   * prime generation            Sources/HomomorphicEncryption/Scalar.swift:113-154
//   * Miller-Rabin                Sources/HomomorphicEncryption/Scalar.swift:160-202
//   * modular inverse             Sources/HomomorphicEncryption/Scalar.swift:76-96
//   * minimal primitive 2N-th root PolyRq/PolyRq+Ntt.swift:87-105
// but is an independent implementation (exact 128-bit `%` arithmetic, deterministic root search); the parity
// tests compare its outputs with the oracle's.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

namespace hecuda {
namespace host {

typedef unsigned long long u64;
typedef unsigned __int128 u128;

inline u64 mulmod(u64 a, u64 b, u64 p) { return (u64)((u128)a * b % p); }

inline u64 powmod(u64 b, u64 e, u64 p) {
    u64 r = 1 % p;
    b %= p;
    for (; e; e >>= 1) {
        if (e & 1) r = mulmod(r, b, p);
        b = mulmod(b, b, p);
    }
    return r;
}

// a^{-1} mod m for gcd(a, m) = 1 (m need not be prime: m~ = 2^32 is a modulus of the BEHZ base). 0 on failure.
inline u64 invmod(u64 a, u64 m) {
    if (m == 0) return 0;
    a %= m;
    if (a == 0) return m == 1 ? 0 : 0;
    __int128 r0 = m, r1 = a, s0 = 0, s1 = 1;
    while (r1 != 0) {
        __int128 q = r0 / r1;
        __int128 t = r0 - q * r1; r0 = r1; r1 = t;
        t = s0 - q * s1; s0 = s1; s1 = t;
    }
    if (r0 != 1) return 0;
    if (s0 < 0) s0 += m;
    return (u64)s0;
}

inline bool is_prime(u64 n) {
    static const u64 witnesses[12] = {2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37};  // deterministic for n < 2^64
    if (n < 2) return false;
    for (u64 w : witnesses) {
        if (n == w) return true;
        if (n % w == 0) return false;
    }
    u64 d = n - 1;
    int r = 0;
    while (!(d & 1)) { d >>= 1; ++r; }
    for (u64 w : witnesses) {
        u64 x = powmod(w, d, n);
        if (x == 1 || x == n - 1) continue;
        bool composite = true;
        for (int i = 1; i < r && composite; ++i) {
            x = mulmod(x, x, n);
            if (x == n - 1) composite = false;
        }
        if (composite) return false;
    }
    return true;
}

// The `count` smallest `bits`-bit primes congruent to 1 mod 2*degree, ascending (RnsTool.swift:30-33 uses this
// with bits = 61 for the BEHZ base Bsk).
inline std::vector<u64> smallest_ntt_primes(int bits, int count, u64 degree) {
    std::vector<u64> out;
    const u64 step = 2 * degree;
    const u64 lo = 1ull << (bits - 1), hi = (bits == 64) ? ~0ull : (1ull << bits);
    for (u64 c = lo + 1; c < hi && (int)out.size() < count; c += step)
        if (c % step == 1 && is_prime(c)) out.push_back(c);
    return out;
}

// Smallest primitive `order`-th root of unity mod prime p (order a power of two dividing p-1); 0 if none.
inline u64 min_primitive_root(u64 order, u64 p) {
    if (order < 2 || (order & (order - 1)) || (p - 1) % order) return 0;
    u64 gen = 0;
    for (u64 g = 2; g < p; ++g) {
        u64 r = powmod(g, (p - 1) / order, p);
        if (powmod(r, order / 2, p) == p - 1) { gen = r; break; }
    }
    if (!gen) return 0;
    // the primitive roots are gen^k for odd k; take the least
    u64 best = gen, cur = gen, g2 = mulmod(gen, gen, p);
    for (u64 k = 1; k < order; k += 2) {
        if (cur < best) best = cur;
        cur = mulmod(cur, g2, p);
    }
    return best;
}

inline unsigned bitrev(unsigned x, int bits) {
    unsigned r = 0;
    for (int i = 0; i < bits; ++i) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
}

inline int bit_length(u64 x) { return x ? 64 - __builtin_clzll(x) : 0; }

// product of moduli mod p
inline u64 prod_mod(const u64 *m, int n, u64 p) {
    u64 r = 1 % p;
    for (int i = 0; i < n; ++i) r = mulmod(r, m[i] % p, p);
    return r;
}
// product of moduli except index `skip`, mod p
inline u64 punctured_mod(const u64 *m, int n, int skip, u64 p) {
    u64 r = 1 % p;
    for (int i = 0; i < n; ++i)
        if (i != skip) r = mulmod(r, m[i] % p, p);
    return r;
}
inline u64 shoup_factor(u64 w, u64 p) { return (u64)(((u128)w << 64) / p); }

// x (w little-endian words) as a double, rounded to nearest with ties to even, like Double(_:) of a wide integer (the
// noise budget's infinity norm, Bfv+Decrypt.swift:137-146).  The leading 64 bits convert with one rounding; every bit
// below them only decides ties, so it is folded into bit 0, far below the rounding bit of the 53-bit result.
inline double wide_to_double(const u64 *x, int w) {
    int top = w - 1;
    while (top >= 0 && !x[top]) --top;
    if (top < 0) return 0.0;
    if (top == 0) return (double)x[0];
    const int lz = __builtin_clzll(x[top]);
    u64 m = lz ? (x[top] << lz) | (x[top - 1] >> (64 - lz)) : x[top];  // the leading 64 bits
    bool sticky = lz ? (x[top - 1] << lz) != 0 : x[top - 1] != 0;      // the bits of x[top - 1] below them
    for (int i = top - 2; i >= 0 && !sticky; --i) sticky = x[i] != 0;
    if (sticky) m |= 1;
    return std::ldexp((double)m, 64 * top - lz);
}

}  // namespace host
}  // namespace hecuda
