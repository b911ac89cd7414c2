// p384.cuh -- the P-384 field and group (SEC 2, FIPS 186-5) as __host__ __device__ functions, for symmetric_pir.cu's
// OPRF evaluation and OPRF server and oprf_client.cu's OPRF client; tests/emu replays them against
// oracle/oprf_oracle.py.
//
//   Field   12 x 32-bit little-endian limbs in Montgomery form, R = 2^384.  p = 2^384 - 2^128 - 2^96 + 2^32 - 1 is
//           -1 mod 2^32, so the per-word Montgomery factor -p^-1 mod 2^32 is 1 and each reduction step's multiplier
//           is the low word itself.  Every function returns a value below p.
//   Scalars mod n through the same Montgomery code with n's own factor -n^-1 mod 2^32 (ModN), kept as plain integers.
//   Group   Jacobian coordinates (x = X/Z^2, y = Y/Z^3, the identity has Z = 0), a = -3 doubling (dbl-2001-b) and
//           the general addition (add-2007-bl).
//   Hashing RFC 9380 P384_XMD:SHA-384_SSWU_RO_: expand_message_xmd with SHA-384, hash_to_field (L = 72, count 2),
//           the straight-line simplified SWU of its appendix F.2 with Z = -12 and sqrt_ratio for p = 3 mod 4, and the
//           sum of the two mapped points (cofactor 1).
//   Scalar  k * P over 96 signed odd 4-bit digits (recode_scalar): a fixed sequence of 4 doublings and one table
//           addition per digit.  scalar_mul indexes the table directly, for the key every thread shares (recoded
//           once on the host) and for public scalars; scalar_mul_ct reads it without secret-dependent addresses or
//           branches, for a secret scalar of one thread.
//   VOPRF   RFC 9497 BlindEvaluate with the DLEQ proof over one element (blind_evaluate_composite, generate_proof),
//           and the client's Blind, VerifyProof and Finalize (blind, verify_proof, unblind_finalize).
#pragma once
#include <cstdint>

#include "sha512.cuh"

#ifdef __CUDACC__
#define P384_HD __host__ __device__ __forceinline__
#else
#define P384_HD inline
#endif

namespace hecuda {
namespace p384 {

constexpr int kLimbs = 12, kDigits = 96, kWindow = 4, kTable = 8;  // table: 1P, 3P, ..., 15P
constexpr int kScalarBytes = 48, kElementBytes = 49, kOutputBytes = 48;

// RFC 9497's contextString for VOPRF mode over P384-SHA384: "OPRFV1-" || I2OSP(0x01, 1) || "-P384-SHA384".  It follows
// the RFC's text; no swift-crypto vector pins these bytes.  HashToGroup's DST is "HashToGroup-" || contextString.
#define HECUDA_OPRF_CONTEXT_STRING "OPRFV1-\x01-P384-SHA384"
#define HECUDA_OPRF_HASH_TO_GROUP_DST "HashToGroup-" HECUDA_OPRF_CONTEXT_STRING
constexpr int kHashToGroupDstBytes = (int)sizeof(HECUDA_OPRF_HASH_TO_GROUP_DST) - 1;  // 32

struct Fe {
    uint32_t v[kLimbs];
};
struct Point {
    Fe x, y, z;
};

#define HECUDA_P384_CONSTANTS(X)                                                                                          \
    X(kP, 0xffffffffu, 0x00000000u, 0x00000000u, 0xffffffffu, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0xffffffffu,     \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)                                                              \
    X(kN, 0xccc52973u, 0xecec196au, 0x48b0a77au, 0x581a0db2u, 0xf4372ddfu, 0xc7634d81u, 0xffffffffu, 0xffffffffu,      \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)                                                              \
    X(kOne, 0x00000001u, 0xffffffffu, 0xffffffffu, 0x00000000u, 0x00000001u, 0x00000000u, 0x00000000u, 0x00000000u,    \
      0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u)                                                              \
    X(kR2, 0x00000001u, 0xfffffffeu, 0x00000000u, 0x00000002u, 0x00000000u, 0xfffffffeu, 0x00000000u, 0x00000002u,     \
      0x00000001u, 0x00000000u, 0x00000000u, 0x00000000u)                                                              \
    X(kR3, 0x00000002u, 0xfffffffcu, 0x00000002u, 0x00000003u, 0xfffffffeu, 0xfffffffcu, 0x00000005u, 0x00000003u,     \
      0xfffffffdu, 0xfffffffdu, 0x00000002u, 0x00000003u)                                                              \
    X(kB, 0x9d412dccu, 0x08118871u, 0x7a4c32ecu, 0xf729add8u, 0x1920022eu, 0x77f2209bu, 0x94938ae2u, 0xe3374beeu,      \
      0x1f022094u, 0xb62b21f4u, 0x604fbff9u, 0xcd08114bu)                                                              \
    X(kA, 0xfffffffcu, 0x00000003u, 0x00000000u, 0xfffffffcu, 0xfffffffbu, 0xffffffffu, 0xffffffffu, 0xffffffffu,      \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)                                                              \
    X(kZ, 0xfffffff3u, 0x0000000cu, 0x00000000u, 0xfffffff3u, 0xfffffff2u, 0xffffffffu, 0xffffffffu, 0xffffffffu,      \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)                                                              \
    X(kSqrtMinusZ, 0xc0a3f1f8u, 0x1cdf6f1cu, 0x4c08f647u, 0xfdf2313bu, 0xd4183d32u, 0x89cb6776u, 0x476b11b6u,          \
      0xacb3a761u, 0xc093fceau, 0xe428a383u, 0x3ae40b98u, 0xd78fa36bu)                                                 \
    X(kGx, 0x49c0b528u, 0x3dd07566u, 0xa0d6ce38u, 0x20e378e2u, 0x541b4d6eu, 0x879c3afcu, 0x59a30effu, 0x64548684u,     \
      0x614ede2bu, 0x812ff723u, 0x299e1513u, 0x4d3aadc2u)                                                              \
    X(kGy, 0x4b03a4feu, 0x23043dadu, 0x7bb4a9acu, 0xa1bfa8bfu, 0x2e83b050u, 0x8bade756u, 0x68f4ffd9u, 0xc6c35219u,     \
      0x3969a840u, 0xdd800226u, 0x5a15c5e9u, 0x2b78abc2u)                                                              \
    X(kPMinus2, 0xfffffffdu, 0x00000000u, 0x00000000u, 0xffffffffu, 0xfffffffeu, 0xffffffffu, 0xffffffffu,             \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)                                                 \
    X(kSqrtRatioC1, 0x3fffffffu, 0x00000000u, 0xc0000000u, 0xbfffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu,         \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu)                                                 \
    X(kSqrtExp, 0x40000000u, 0x00000000u, 0xc0000000u, 0xbfffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu,             \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu)                                                 \
    X(kNR2, 0x19b409a9u, 0x2d319b24u, 0xdf1aa419u, 0xff3d81e5u, 0xfcb82947u, 0xbc3e483au, 0x4aab1cc5u, 0xd40d4917u,    \
      0x28266895u, 0x3fb05b7au, 0x2b39bf21u, 0x0c84ee01u)                                                              \
    X(kNOne, 0x333ad68du, 0x1313e695u, 0xb74f5885u, 0xa7e5f24du, 0x0bc8d220u, 0x389cb27eu, 0x00000000u, 0x00000000u,   \
      0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u)                                                              \
    X(kNMinus2, 0xccc52971u, 0xecec196au, 0x48b0a77au, 0x581a0db2u, 0xf4372ddfu, 0xc7634d81u, 0xffffffffu,             \
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu)
// p and n are plain integers; kOne .. kGy are in Montgomery form (x R mod p): R, R^2, R^3, b, a = -3, Z = -12,
// sqrt(-Z) = sqrt(12) and the generator; kPMinus2, kSqrtRatioC1 = (p - 3) / 4 and kSqrtExp = (p + 1) / 4 are
// exponents; kNR2 = R^2 mod n and kNOne = R mod n; kNMinus2 = n - 2 is an exponent.

#ifdef __CUDACC__
#define HECUDA_P384_DEVICE(name, ...) static __constant__ Fe name##Device = {{__VA_ARGS__}};
HECUDA_P384_CONSTANTS(HECUDA_P384_DEVICE)
#undef HECUDA_P384_DEVICE
#endif
#define HECUDA_P384_HOST(name, ...) static const Fe name##Host = {{__VA_ARGS__}};
HECUDA_P384_CONSTANTS(HECUDA_P384_HOST)
#undef HECUDA_P384_HOST

#ifdef __CUDA_ARCH__
#define P384_CONST(name) name##Device
#else
#define P384_CONST(name) name##Host
#endif

// ---------------------------------------------------------------- field and scalars
// The two moduli share one Montgomery code: ModP for the field, ModN for scalars mod the group order.  kM0 is the
// per-word factor -m^-1 mod 2^32; it is 1 for p, so p's reduction step multiplies by the low word itself.
// one() is R mod m, the Montgomery form of 1.
struct ModP {
    static constexpr uint32_t kM0 = 1;
    P384_HD static const Fe &m() { return P384_CONST(kP); }
    P384_HD static const Fe &one() { return P384_CONST(kOne); }
};
struct ModN {
    static constexpr uint32_t kM0 = 0xe88fdc45u;
    P384_HD static const Fe &m() { return P384_CONST(kN); }
    P384_HD static const Fe &one() { return P384_CONST(kNOne); }
};

// r = t - m if t (with carry word `top`) >= m, else t
template <class M>
P384_HD void reduce_once(Fe &r, const uint32_t t[kLimbs], uint32_t top) {
    const Fe &p = M::m();
    uint32_t d[kLimbs];
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) {
        const uint64_t s = (uint64_t)t[i] - p.v[i] - borrow;
        d[i] = (uint32_t)s;
        borrow = (s >> 32) & 1;
    }
    const uint32_t keep = (uint32_t)0 - (uint32_t)(borrow & (uint64_t)(top == 0));  // all ones: t < m
    for (int i = 0; i < kLimbs; ++i) r.v[i] = (t[i] & keep) | (d[i] & ~keep);
}

// a + b mod m for a, b < m
template <class M>
P384_HD void add(Fe &r, const Fe &a, const Fe &b) {
    uint32_t t[kLimbs];
    uint64_t c = 0;
    for (int i = 0; i < kLimbs; ++i) {
        c += (uint64_t)a.v[i] + b.v[i];
        t[i] = (uint32_t)c;
        c >>= 32;
    }
    reduce_once<M>(r, t, (uint32_t)c);
}
P384_HD void add(Fe &r, const Fe &a, const Fe &b) { add<ModP>(r, a, b); }

// a - b mod m for a, b < m
template <class M>
P384_HD void sub(Fe &r, const Fe &a, const Fe &b) {
    const Fe &p = M::m();
    uint32_t t[kLimbs];
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) {
        const uint64_t s = (uint64_t)a.v[i] - b.v[i] - borrow;
        t[i] = (uint32_t)s;
        borrow = (s >> 32) & 1;
    }
    const uint32_t mask = (uint32_t)0 - (uint32_t)borrow;  // add m back after a borrow
    uint64_t c = 0;
    for (int i = 0; i < kLimbs; ++i) {
        c += (uint64_t)t[i] + (p.v[i] & mask);
        r.v[i] = (uint32_t)c;
        c >>= 32;
    }
}
P384_HD void sub(Fe &r, const Fe &a, const Fe &b) { sub<ModP>(r, a, b); }

P384_HD void neg(Fe &r, const Fe &a) {
    Fe zero = {};
    sub(r, zero, a);
}

// a b R^-1 mod m by CIOS; a may be any value below 2^384 and b below m
template <class M>
P384_HD void mul(Fe &r, const Fe &a, const Fe &b) {
    const Fe &p = M::m();
    uint32_t t[kLimbs + 2] = {};
    for (int i = 0; i < kLimbs; ++i) {
        const uint32_t bi = b.v[i];
        uint64_t c = 0;
        for (int j = 0; j < kLimbs; ++j) {
            c = (uint64_t)a.v[j] * bi + t[j] + (c >> 32);
            t[j] = (uint32_t)c;
        }
        c = (uint64_t)t[kLimbs] + (c >> 32);
        t[kLimbs] = (uint32_t)c;
        t[kLimbs + 1] = (uint32_t)(c >> 32);
        const uint32_t m = t[0] * M::kM0;
        c = (uint64_t)m * p.v[0] + t[0];
        for (int j = 1; j < kLimbs; ++j) {
            c = (uint64_t)m * p.v[j] + t[j] + (c >> 32);
            t[j - 1] = (uint32_t)c;
        }
        c = (uint64_t)t[kLimbs] + (c >> 32);
        t[kLimbs - 1] = (uint32_t)c;
        t[kLimbs] = t[kLimbs + 1] + (uint32_t)(c >> 32);
    }
    reduce_once<M>(r, t, t[kLimbs]);
}
P384_HD void mul(Fe &r, const Fe &a, const Fe &b) { mul<ModP>(r, a, b); }

P384_HD void sqr(Fe &r, const Fe &a) { mul(r, a, a); }

P384_HD bool is_zero(const Fe &a) {
    uint32_t acc = 0;
    for (int i = 0; i < kLimbs; ++i) acc |= a.v[i];
    return acc == 0;
}

P384_HD bool equal(const Fe &a, const Fe &b) {
    uint32_t acc = 0;
    for (int i = 0; i < kLimbs; ++i) acc |= a.v[i] ^ b.v[i];
    return acc == 0;
}

// r = c ? a : b
P384_HD void select(Fe &r, bool c, const Fe &a, const Fe &b) {
    const uint32_t m = (uint32_t)0 - (uint32_t)c;
    for (int i = 0; i < kLimbs; ++i) r.v[i] = (a.v[i] & m) | (b.v[i] & ~m);
}

P384_HD void to_mont(Fe &r, const Fe &a) { mul(r, a, P384_CONST(kR2)); }
P384_HD void from_mont(Fe &r, const Fe &a) {
    Fe one = {};
    one.v[0] = 1;
    mul(r, a, one);
}

// a^e mod m for a in Montgomery form and a public exponent e (a plain integer), by fixed 4-bit windows.  Only the
// exponent's digits choose a branch or a table entry, so a may be secret.
template <class M>
P384_HD void pow_fixed(Fe &r, const Fe &a, const Fe &e) {
    Fe table[16];
    table[0] = M::one();
    table[1] = a;
    for (int i = 2; i < 16; ++i) mul<M>(table[i], table[i - 1], a);
    r = M::one();
    for (int w = kDigits - 1; w >= 0; --w) {
        for (int s = 0; s < 4; ++s) mul<M>(r, r, r);
        const uint32_t nibble = (e.v[w >> 3] >> (4 * (w & 7))) & 15;
        if (nibble) mul<M>(r, r, table[nibble]);
    }
}
P384_HD void pow_fixed(Fe &r, const Fe &a, const Fe &e) { pow_fixed<ModP>(r, a, e); }

P384_HD void inv(Fe &r, const Fe &a) { pow_fixed(r, a, P384_CONST(kPMinus2)); }

// RFC 9380 F.2.1.2, q = 3 mod 4: returns whether u/v is square, y = sqrt(u/v) if so, else sqrt(Z u/v)
P384_HD bool sqrt_ratio(Fe &y, const Fe &u, const Fe &v) {
    Fe tv1, tv2, y1, y2, tv3;
    sqr(tv1, v);
    mul(tv2, u, v);
    mul(tv1, tv1, tv2);
    pow_fixed(y1, tv1, P384_CONST(kSqrtRatioC1));
    mul(y1, y1, tv2);
    mul(y2, y1, P384_CONST(kSqrtMinusZ));
    sqr(tv3, y1);
    mul(tv3, tv3, v);
    const bool is_qr = equal(tv3, u);
    select(y, is_qr, y1, y2);
    return is_qr;
}

P384_HD bool is_square(const Fe &a) {
    Fe y;
    return sqrt_ratio(y, a, P384_CONST(kOne));
}

P384_HD uint32_t sgn0(const Fe &a) {
    Fe plain;
    from_mont(plain, a);
    return plain.v[0] & 1;
}

// 48 big-endian bytes <-> a plain integer (not reduced)
P384_HD void from_bytes(Fe &r, const unsigned char *be) {
    for (int i = 0; i < kLimbs; ++i) {
        const unsigned char *q = be + 4 * (kLimbs - 1 - i);
        r.v[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    }
}
P384_HD void to_bytes(unsigned char *be, const Fe &a) {
    for (int i = 0; i < kScalarBytes; ++i) be[i] = (unsigned char)(a.v[kLimbs - 1 - i / 4] >> (24 - 8 * (i & 3)));
}

// A 72-byte big-endian integer as hi 2^384 + lo
P384_HD void split_bytes72(Fe &hi, Fe &lo, const unsigned char be[72]) {
    hi = Fe{};
    for (int i = 0; i < 6; ++i) {
        const unsigned char *q = be + 4 * (5 - i);
        hi.v[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    }
    from_bytes(lo, be + 24);
}

// A 72-byte big-endian integer mod p, in Montgomery form: hi 2^384 + lo -> hi R^3 R^-1 + lo R^2 R^-1 = (hi 2^384 + lo) R
P384_HD void from_bytes72(Fe &r, const unsigned char be[72]) {
    Fe hi, lo, a, b;
    split_bytes72(hi, lo, be);
    mul(a, hi, P384_CONST(kR3));
    mul(b, lo, P384_CONST(kR2));
    add(r, a, b);
}

// The same integer mod n as a plain integer (HashToScalar's reduction): hi R^2 R^-1 = hi 2^384 mod n, and lo < 2^384 <
// 2n needs one conditional subtraction
P384_HD void from_bytes72_mod_n(Fe &r, const unsigned char be[72]) {
    Fe hi, lo, a, b;
    split_bytes72(hi, lo, be);
    mul<ModN>(a, hi, P384_CONST(kNR2));
    reduce_once<ModN>(b, lo.v, 0);
    add<ModN>(r, a, b);
}

// a b mod n for plain a < 2^384 and b < n: (a R^2 R^-1) b R^-1
P384_HD void mul_mod_n(Fe &r, const Fe &a, const Fe &b) {
    Fe t;
    mul<ModN>(t, a, P384_CONST(kNR2));
    mul<ModN>(r, t, b);
}

// a^-1 mod n for a plain a in [1, n - 1] (0 for a = 0), as a^(n - 2) (Fermat) in Montgomery form: a R -> a^-1 R -> a^-1.
// a may be secret: pow_fixed branches on the public exponent only.
P384_HD void inv_mod_n(Fe &r, const Fe &a) {
    Fe am, t, one = {};
    one.v[0] = 1;
    mul<ModN>(am, a, P384_CONST(kNR2));
    pow_fixed<ModN>(t, am, P384_CONST(kNMinus2));
    mul<ModN>(r, t, one);
}

// a < b for plain integers, without a branch
P384_HD bool less_than(const Fe &a, const Fe &b) {
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) borrow = (((uint64_t)a.v[i] - b.v[i] - borrow) >> 32) & 1;
    return borrow != 0;
}

// ---------------------------------------------------------------- group
P384_HD bool is_identity(const Point &p) { return is_zero(p.z); }

// dbl-2001-b (a = -3)
P384_HD void dbl(Point &r, const Point &p) {
    Fe delta, gamma, beta, alpha, t0, t1;
    sqr(delta, p.z);
    sqr(gamma, p.y);
    mul(beta, p.x, gamma);
    sub(t0, p.x, delta);
    add(t1, p.x, delta);
    mul(alpha, t0, t1);
    add(t0, alpha, alpha);
    add(alpha, t0, alpha);  // 3 (x - delta)(x + delta)
    add(t0, p.y, p.z);
    sqr(t0, t0);
    sub(t0, t0, gamma);
    sub(r.z, t0, delta);
    add(t1, beta, beta);
    add(t1, t1, t1);  // 4 beta
    add(t0, t1, t1);  // 8 beta
    sqr(r.x, alpha);
    sub(r.x, r.x, t0);
    sub(t1, t1, r.x);
    mul(t1, alpha, t1);
    sqr(gamma, gamma);
    add(gamma, gamma, gamma);
    add(gamma, gamma, gamma);
    add(gamma, gamma, gamma);  // 8 gamma^2
    sub(r.y, t1, gamma);
}

// add-2007-bl.  Equal inputs fall back to the doubling, opposite ones give the identity.
P384_HD void add(Point &r, const Point &p, const Point &q) {
    if (is_identity(p)) {
        r = q;
        return;
    }
    if (is_identity(q)) {
        r = p;
        return;
    }
    Fe z1z1, z2z2, u1, u2, s1, s2, h, i, j, rr, v, t;
    sqr(z1z1, p.z);
    sqr(z2z2, q.z);
    mul(u1, p.x, z2z2);
    mul(u2, q.x, z1z1);
    mul(s1, p.y, q.z);
    mul(s1, s1, z2z2);
    mul(s2, q.y, p.z);
    mul(s2, s2, z1z1);
    sub(h, u2, u1);
    sub(rr, s2, s1);
    add(rr, rr, rr);
    if (is_zero(h)) {
        if (is_zero(rr)) {
            dbl(r, p);
        } else {
            r.x = P384_CONST(kOne), r.y = P384_CONST(kOne), r.z = Fe{};
        }
        return;
    }
    add(i, h, h);
    sqr(i, i);
    mul(j, h, i);
    mul(v, u1, i);
    Fe x3, y3;
    sqr(x3, rr);
    sub(x3, x3, j);
    sub(x3, x3, v);
    sub(x3, x3, v);
    sub(t, v, x3);
    mul(y3, rr, t);
    mul(t, s1, j);
    add(t, t, t);
    sub(y3, y3, t);
    add(t, p.z, q.z);
    sqr(t, t);
    sub(t, t, z1z1);
    sub(t, t, z2z2);
    mul(r.z, t, h);
    r.x = x3, r.y = y3;
}

// (x, y) with x, y in Montgomery form; false for the identity
P384_HD bool to_affine(Fe &x, Fe &y, const Point &p) {
    if (is_identity(p)) return false;
    Fe zi, zi2;
    inv(zi, p.z);
    sqr(zi2, zi);
    mul(x, p.x, zi2);
    mul(zi2, zi2, zi);
    mul(y, p.y, zi2);
    return true;
}

// SEC1 compressed encoding, 49 bytes (RFC 9497 SerializeElement); the identity (never produced by a valid key and a
// hashed input, except with negligible probability) encodes as 49 zero bytes
P384_HD void compress_affine(unsigned char out[kElementBytes], const Fe &x, const Fe &y) {
    Fe xp, yp;
    from_mont(xp, x);
    from_mont(yp, y);
    out[0] = (unsigned char)(2 | (yp.v[0] & 1));
    to_bytes(out + 1, xp);
}

P384_HD void compress(unsigned char out[kElementBytes], const Point &p) {
    Fe x, y;
    if (!to_affine(x, y, p)) {
        for (int i = 0; i < kElementBytes; ++i) out[i] = 0;
        return;
    }
    compress_affine(out, x, y);
}

// RFC 9497 DeserializeElement: SEC1 compressed with prefix 2 or 3, x < p and x^3 - 3x + b a square; false otherwise.
// The encoding is public, so this branches on it.  r = (x, y, 1) in Montgomery form.
P384_HD bool decompress(Point &r, const unsigned char in[kElementBytes]) {
    if (in[0] != 2 && in[0] != 3) return false;
    Fe x, y2, y, t;
    from_bytes(x, in + 1);
    if (!less_than(x, P384_CONST(kP))) return false;
    to_mont(r.x, x);
    sqr(t, r.x);
    add(t, t, P384_CONST(kA));
    mul(y2, t, r.x);
    add(y2, y2, P384_CONST(kB));
    pow_fixed(y, y2, P384_CONST(kSqrtExp));  // p = 3 mod 4
    sqr(t, y);
    if (!equal(t, y2)) return false;
    from_mont(t, y);
    if ((t.v[0] & 1) != (in[0] & 1u)) neg(y, y);  // y = 0 has no point: the group's order is odd
    r.y = y, r.z = P384_CONST(kOne);
    return true;
}

// ---------------------------------------------------------------- hash to curve
// RFC 9380 6.6.2 simplified SWU (straight-line, F.2), with the final division kept as the Jacobian Z: the result is
// (x_num tv4, y tv4^3, tv4) for x = x_num / tv4
P384_HD bool map_to_curve(Point &r, const Fe &u) {
    Fe tv1, tv2, tv3, tv4, tv5, tv6, x, y, y1, t;
    sqr(tv1, u);
    mul(tv1, P384_CONST(kZ), tv1);
    sqr(tv2, tv1);
    add(tv2, tv2, tv1);
    add(tv3, tv2, P384_CONST(kOne));
    mul(tv3, P384_CONST(kB), tv3);
    neg(t, tv2);
    select(tv4, !is_zero(tv2), t, P384_CONST(kZ));
    mul(tv4, P384_CONST(kA), tv4);
    sqr(tv2, tv3);
    sqr(tv6, tv4);
    mul(tv5, P384_CONST(kA), tv6);
    add(tv2, tv2, tv5);
    mul(tv2, tv2, tv3);
    mul(tv6, tv6, tv4);
    mul(tv5, P384_CONST(kB), tv6);
    add(tv2, tv2, tv5);
    mul(x, tv1, tv3);
    const bool gx1_square = sqrt_ratio(y1, tv2, tv6);
    mul(y, tv1, u);
    mul(y, y, y1);
    select(x, gx1_square, tv3, x);
    select(y, gx1_square, y1, y);
    neg(t, y);
    select(y, sgn0(u) == sgn0(y), y, t);
    mul(r.x, x, tv4);
    sqr(t, tv4);
    mul(t, t, tv4);
    mul(r.y, y, t);
    r.z = tv4;
    return gx1_square;
}

// expand_message_xmd(msg, DST, len_in_bytes) with SHA-384 (RFC 9380 5.3.1), in two halves so that a caller can stream
// msg into the hasher: xmd_begin absorbs Z_pad, the caller absorbs msg, xmd_finish writes len_in_bytes (<= 255 * 48)
// bytes to out.  DST is at most 255 bytes.
P384_HD void xmd_begin(sha512::Sha384 &s) {
    s.init();
    s.zeros(128);  // Z_pad
}

P384_HD void xmd_finish(unsigned char *out, int len_in_bytes, sha512::Sha384 &s, const char *dst_chars, int dst_len) {
    const unsigned char *dst = (const unsigned char *)dst_chars;
    s.byte((uint32_t)len_in_bytes >> 8), s.byte((uint32_t)len_in_bytes), s.byte(0);  // I2OSP(len, 2) || I2OSP(0, 1)
    s.bytes(dst, dst_len), s.byte((uint32_t)dst_len);
    unsigned char b0[48], bi[48];
    s.finish(b0);
    for (int i = 1; 48 * (i - 1) < len_in_bytes; ++i) {
        s.init();
        for (int j = 0; j < 48; ++j) s.byte(i == 1 ? b0[j] : (unsigned char)(b0[j] ^ bi[j]));
        s.byte((uint32_t)i);
        s.bytes(dst, dst_len), s.byte((uint32_t)dst_len);
        s.finish(bi);
        for (int j = 0; j < 48 && 48 * (i - 1) + j < len_in_bytes; ++j) out[48 * (i - 1) + j] = bi[j];
    }
}

P384_HD void expand_message_xmd(unsigned char *out, int len_in_bytes, const unsigned char *msg, long long len,
                                const char *dst, int dst_len) {
    sha512::Sha384 s;
    xmd_begin(s);
    s.bytes(msg, len);
    xmd_finish(out, len_in_bytes, s, dst, dst_len);
}

// HashToGroup(msg): hash_to_field (two 72-byte field elements), map both, add
P384_HD void hash_to_group(Point &r, const unsigned char *msg, long long len) {
    unsigned char uniform[144];
    expand_message_xmd(uniform, 144, msg, len, HECUDA_OPRF_HASH_TO_GROUP_DST, kHashToGroupDstBytes);
    Fe u0, u1;
    from_bytes72(u0, uniform);
    from_bytes72(u1, uniform + 72);
    Point q0, q1;
    map_to_curve(q0, u0);
    map_to_curve(q1, u1);
    add(r, q0, q1);
}

// ---------------------------------------------------------------- scalar multiplication
// 0 < k < n for a plain 384-bit k
P384_HD bool scalar_valid(const Fe &k) { return !is_zero(k) && less_than(k, P384_CONST(kN)); }

// The recoding of a k in [0, n - 1]: k is made odd (k' = n - k and flip = 1 when k is even, since n is odd), then
// k' = sum d_i 16^i with 96 odd digits |d_i| <= 15, d_95 > 0 (regular signed windows).  digits[96] = flip.  No branch
// or address depends on k, so a thread can recode its own secret scalar; the shared key is recoded once on the host.
P384_HD void recode_scalar(const Fe &k, signed char digits[kDigits + 1]) {
    const Fe &n = P384_CONST(kN);
    Fe w, nk;
    const uint32_t flip = (k.v[0] & 1) ^ 1;
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) {
        const uint64_t s = (uint64_t)n.v[i] - k.v[i] - borrow;
        nk.v[i] = (uint32_t)s;
        borrow = (s >> 32) & 1;
    }
    select(w, flip != 0, nk, k);
    for (int d = 0; d < kDigits - 1; ++d) {
        const int digit = (int)(w.v[0] & 31) - 16;
        digits[d] = (signed char)digit;
        // w = (w - digit) >> 4; w - digit is 16 mod 32, so the shift is exact
        int64_t c = -digit;  // signed carry: -1, 0 or 1 after each limb
        for (int i = 0; i < kLimbs; ++i) {
            c += w.v[i];
            w.v[i] = (uint32_t)c;
            c >>= 32;
        }
        for (int i = 0; i < kLimbs; ++i) w.v[i] = (w.v[i] >> 4) | (i + 1 < kLimbs ? w.v[i + 1] << 28 : 0);
    }
    digits[kDigits - 1] = (signed char)w.v[0];
    digits[kDigits] = (signed char)flip;
}

// k P from the recoding: P, 3P, ..., 15P, then from the top digit down 4 doublings and the addition of +-|d| P.  The
// only branch that depends on k is add()'s equal-inputs case, which a few keys reach at their last digit (k = n - 6,
// for instance) and which every row of a launch then takes together, since it depends on k alone.
P384_HD void scalar_mul(Point &r, const Point &p, const signed char *digits) {
    Point table[kTable], twice;
    table[0] = p;
    dbl(twice, p);
    for (int i = 1; i < kTable; ++i) add(table[i], table[i - 1], twice);
    Point acc = table[(digits[kDigits - 1] - 1) >> 1];
    for (int d = kDigits - 2; d >= 0; --d) {
        for (int s = 0; s < kWindow; ++s) dbl(acc, acc);
        const int digit = digits[d];
        const int magnitude = digit < 0 ? -digit : digit;
        Point q = table[(magnitude - 1) >> 1];
        Fe ny;
        neg(ny, q.y);
        select(q.y, digit < 0, ny, q.y);
        add(acc, acc, q);
    }
    Fe ny;
    neg(ny, acc.y);
    select(acc.y, digits[kDigits] != 0, ny, acc.y);
    r = acc;
}

// q = sign(digit) table[(|digit| - 1) / 2] for an odd digit, reading all eight entries and negating with a mask
P384_HD void lookup_ct(Point &q, const Point table[kTable], int digit) {
    const int sign = digit >> 31;  // -1 or 0
    const int index = (((digit ^ sign) - sign) - 1) >> 1;
    q = table[0];
    for (int i = 1; i < kTable; ++i) {
        const bool hit = i == index;
        select(q.x, hit, table[i].x, q.x);
        select(q.y, hit, table[i].y, q.y);
        select(q.z, hit, table[i].z, q.z);
    }
    Fe ny;
    neg(ny, q.y);
    select(q.y, sign != 0, ny, q.y);
}

// k P for a secret scalar of this thread alone (the proof nonce), recoded on the device: scalar_mul's operation
// sequence, with every table read through lookup_ct and the final flip applied with a mask, so no branch and no memory
// address depends on k.  add()'s identity and equal-inputs branches remain; a uniformly random k reaches them only if
// a partial sum of the ladder is the identity or +-(the entry being added), which has negligible probability.
P384_HD void scalar_mul_ct(Point &r, const Point &p, const signed char digits[kDigits + 1]) {
    Point table[kTable], twice, acc, q;
    table[0] = p;
    dbl(twice, p);
    for (int i = 1; i < kTable; ++i) add(table[i], table[i - 1], twice);
    lookup_ct(acc, table, digits[kDigits - 1]);
    for (int d = kDigits - 2; d >= 0; --d) {
        for (int s = 0; s < kWindow; ++s) dbl(acc, acc);
        lookup_ct(q, table, digits[d]);
        add(acc, acc, q);
    }
    Fe ny;
    neg(ny, acc.y);
    select(acc.y, digits[kDigits] != 0, ny, acc.y);
    r = acc;
}

P384_HD void generator(Point &g) {
    g.x = P384_CONST(kGx), g.y = P384_CONST(kGy), g.z = P384_CONST(kOne);
}

// RFC 9497 Finalize's hash: SHA-384(I2OSP(len, 2) || input || I2OSP(49, 2) || issued || "Finalize"); len < 2^16
P384_HD void finalize_hash(unsigned char out[kOutputBytes], const unsigned char *input, long long len,
                           const unsigned char issued[kElementBytes]) {
    sha512::Sha384 s;
    s.init();
    s.byte((uint32_t)(len >> 8)), s.byte((uint32_t)len);
    s.bytes(input, len);
    s.byte(0), s.byte(kElementBytes);
    s.bytes(issued, kElementBytes);
    s.bytes((const unsigned char *)"Finalize", 8);
    s.finish(out);
}

// RFC 9497 Evaluate's output for one input: finalize_hash of Ser(k HashToGroup(input))
P384_HD void oprf_evaluate(unsigned char out[kOutputBytes], const signed char *digits, const unsigned char *input,
                           long long len) {
    Point e, z;
    hash_to_group(e, input, len);
    scalar_mul(z, e, digits);
    unsigned char issued[kElementBytes];
    compress(issued, z);
    finalize_hash(out, input, len, issued);
}

// ---------------------------------------------------------------- VOPRF BlindEvaluate with the DLEQ proof
// RFC 9497 3.3.2 BlindEvaluate and 2.2.1 GenerateProof with ComputeCompositesFast, for a proof over one element, as
// swift-crypto's P384._VOPRF.PrivateKey.evaluate returns it: Ser(k B) || I2OSP(c, 48) || I2OSP(s, 48).  A query is
// answered in two halves, blind_evaluate_composite then generate_proof, with the composite M passed between them.
#define HECUDA_OPRF_HASH_TO_SCALAR_DST "HashToScalar-" HECUDA_OPRF_CONTEXT_STRING
#define HECUDA_OPRF_SEED_DST "Seed-" HECUDA_OPRF_CONTEXT_STRING
#define HECUDA_OPRF_PROOF_NONCE_DST "HECUDA-ProofNonce-" HECUDA_OPRF_CONTEXT_STRING  // see proof_nonce
constexpr int kHashToScalarDstBytes = (int)sizeof(HECUDA_OPRF_HASH_TO_SCALAR_DST) - 1;  // 33
constexpr int kSeedDstBytes = (int)sizeof(HECUDA_OPRF_SEED_DST) - 1;                    // 25
constexpr int kProofNonceDstBytes = (int)sizeof(HECUDA_OPRF_PROOF_NONCE_DST) - 1;       // 38
constexpr int kSeedBytes = 48, kNonceSeedBytes = 32, kProofBytes = 96;
constexpr int kResponseBytes = kElementBytes + kProofBytes;  // 145

P384_HD void i2osp2(sha512::Sha384 &s, int v) { s.byte((uint32_t)v >> 8), s.byte((uint32_t)v); }

// HashToScalar(msg): hash_to_field(msg, 1) with modulus n, L = 72 and DST "HashToScalar-" || contextString, for a msg
// the caller absorbed after xmd_begin
P384_HD void hash_to_scalar_finish(Fe &r, sha512::Sha384 &s) {
    unsigned char u[72];
    xmd_finish(u, 72, s, HECUDA_OPRF_HASH_TO_SCALAR_DST, kHashToScalarDstBytes);
    from_bytes72_mod_n(r, u);
}

// ComputeCompositesFast's seed for bm = SerializeElement(k G): SHA-384(I2OSP(49, 2) || bm || I2OSP(25, 2) || "Seed-"
// || contextString), the same for every query under one key
P384_HD void composite_seed(unsigned char seed[kSeedBytes], const unsigned char bm[kElementBytes]) {
    sha512::Sha384 s;
    s.init();
    i2osp2(s, kElementBytes);
    s.bytes(bm, kElementBytes);
    i2osp2(s, kSeedDstBytes);
    s.bytes((const unsigned char *)HECUDA_OPRF_SEED_DST, kSeedDstBytes);
    s.finish(seed);
}

// d0 = HashToScalar(I2OSP(48, 2) || seed || I2OSP(0, 2) || I2OSP(49, 2) || Ser(B) || I2OSP(49, 2) || Ser(D) ||
// "Composite")
P384_HD void composite_scalar(Fe &d0, const unsigned char seed[kSeedBytes], const unsigned char blinded[kElementBytes],
                              const unsigned char evaluated[kElementBytes]) {
    sha512::Sha384 s;
    xmd_begin(s);
    i2osp2(s, kSeedBytes);
    s.bytes(seed, kSeedBytes);
    i2osp2(s, 0);
    i2osp2(s, kElementBytes);
    s.bytes(blinded, kElementBytes);
    i2osp2(s, kElementBytes);
    s.bytes(evaluated, kElementBytes);
    s.bytes((const unsigned char *)"Composite", 9);
    hash_to_scalar_finish(d0, s);
}

// The first half: B = DeserializeElement(query), evaluated = Ser(D) with D = k B, and M = d0 B in affine Montgomery
// coordinates (mx, my).  A valid query is its own Ser(B): x < p and the prefix's parity bit make the encoding unique.
// d0 is public, so M uses scalar_mul.  False for an invalid query, and for M the identity (d0 = 0, negligible).
P384_HD bool blind_evaluate_composite(unsigned char evaluated[kElementBytes], Fe &mx, Fe &my,
                                      const unsigned char query[kElementBytes], const signed char *k_digits,
                                      const unsigned char seed[kSeedBytes]) {
    Point b, p;
    if (!decompress(b, query)) return false;
    scalar_mul(p, b, k_digits);
    compress(evaluated, p);
    Fe d0;
    composite_scalar(d0, seed, query, evaluated);
    signed char digits[kDigits + 1];
    recode_scalar(d0, digits);
    scalar_mul(p, b, digits);
    return to_affine(mx, my, p);
}

// The proof nonce r = OS2IP(expand_message_xmd(I2OSP(k, 48) || seed32 || Ser(B), "HECUDA-ProofNonce-" ||
// contextString, 72)) mod n.  RFC 9497 draws r at random, and any r in [1, n - 1] gives a proof that a verifier accepts.
// Reusing one r under two different challenges reveals k = (s1 - s2) / (c2 - c1); deriving r from (k, B), hedged with
// the caller's seed32, makes a repeated seed harmless, since equal (k, B) give equal challenges.
P384_HD void proof_nonce(Fe &r, const Fe &k, const unsigned char seed32[kNonceSeedBytes],
                         const unsigned char query[kElementBytes]) {
    unsigned char kb[kScalarBytes], u[72];
    to_bytes(kb, k);
    sha512::Sha384 s;
    xmd_begin(s);
    s.bytes(kb, kScalarBytes);
    s.bytes(seed32, kNonceSeedBytes);
    s.bytes(query, kElementBytes);
    xmd_finish(u, 72, s, HECUDA_OPRF_PROOF_NONCE_DST, kProofNonceDstBytes);
    from_bytes72_mod_n(r, u);
}

// The second half, GenerateProof: Z = k M, t2 = r G, t3 = r M, c = HashToScalar(I2OSP(49, 2) || bm || I2OSP(49, 2) ||
// Ser(M) || I2OSP(49, 2) || Ser(Z) || I2OSP(49, 2) || Ser(t2) || I2OSP(49, 2) || Ser(t3) || "Challenge") and
// s = r - c k mod n, written as proof = I2OSP(c, 48) || I2OSP(s, 48).  k is plain, in [1, n - 1], with its recoding
// k_digits; r in [1, n - 1] is secret and differs per thread, so t2 and t3 run through scalar_mul_ct.
P384_HD void generate_proof(unsigned char proof[kProofBytes], const signed char *k_digits, const Fe &k,
                            const unsigned char bm[kElementBytes], const Fe &mx, const Fe &my, const Fe &r) {
    sha512::Sha384 s;
    xmd_begin(s);
    unsigned char e[kElementBytes];
    i2osp2(s, kElementBytes);
    s.bytes(bm, kElementBytes);
    compress_affine(e, mx, my);
    i2osp2(s, kElementBytes);
    s.bytes(e, kElementBytes);
    Point m, g, p;
    m.x = mx, m.y = my, m.z = P384_CONST(kOne);
    scalar_mul(p, m, k_digits);
    compress(e, p);
    i2osp2(s, kElementBytes);
    s.bytes(e, kElementBytes);
    signed char digits[kDigits + 1];
    recode_scalar(r, digits);
    generator(g);
    scalar_mul_ct(p, g, digits);
    compress(e, p);
    i2osp2(s, kElementBytes);
    s.bytes(e, kElementBytes);
    scalar_mul_ct(p, m, digits);
    compress(e, p);
    i2osp2(s, kElementBytes);
    s.bytes(e, kElementBytes);
    s.bytes((const unsigned char *)"Challenge", 9);
    Fe c, ck;
    hash_to_scalar_finish(c, s);
    mul_mod_n(ck, c, k);
    sub<ModN>(ck, r, ck);
    to_bytes(proof, c);
    to_bytes(proof + kScalarBytes, ck);
}

// ---------------------------------------------------------------- VOPRF client: Blind, VerifyProof, Finalize
// RFC 9497 3.3.2 for one element, as swift-crypto's P384._VOPRF.PublicKey.blind and .finalize run it.  The blind r is
// the client's secret, so r B and r^-1 D go through scalar_mul_ct and r^-1 through inv_mod_n; the proof's scalars and
// every point of the verification are public, so VerifyProof uses scalar_mul.

// Blind: query = Ser(r HashToGroup(input)) for a plain r in [1, n - 1]
P384_HD void blind(unsigned char query[kElementBytes], const Fe &r, const unsigned char *input, long long len) {
    Point e, b;
    hash_to_group(e, input, len);
    signed char digits[kDigits + 1];
    recode_scalar(r, digits);
    scalar_mul_ct(b, e, digits);
    compress(query, b);
}

// The challenge's element: I2OSP(49, 2) || Ser(p)
P384_HD void absorb_element(sha512::Sha384 &s, const Point &p) {
    unsigned char e[kElementBytes];
    compress(e, p);
    i2osp2(s, kElementBytes);
    s.bytes(e, kElementBytes);
}

// VerifyProof (2.2.2) over one element with ComputeComposites: pk_ser = Ser(pkS) and seed = composite_seed(pk_ser) are
// per key, B and D the decoded query and evaluated element, their encodings `blinded` and `evaluated`, and proof = c ||
// s.  c, s < n; d0 = composite_scalar(seed, Ser(B), Ser(D)); M = d0 B and Z = d0 D; t2 = s G + c pkS and t3 = s M + c Z;
// true when HashToScalar(Ser(pkS), Ser(M), Z, t2, t3 framed || "Challenge") is c.  The six products run through one
// scalar_mul in a loop, so a kernel holds one copy of the ladder.
P384_HD bool verify_proof(const Point &pk, const unsigned char pk_ser[kElementBytes],
                          const unsigned char seed[kSeedBytes], const Point &b, const unsigned char blinded[kElementBytes],
                          const Point &d, const unsigned char evaluated[kElementBytes],
                          const unsigned char proof[kProofBytes]) {
    Fe c, s, d0;
    from_bytes(c, proof);
    from_bytes(s, proof + kScalarBytes);
    if (!less_than(c, P384_CONST(kN)) || !less_than(s, P384_CONST(kN))) return false;
    composite_scalar(d0, seed, blinded, evaluated);
    // products: M = d0 B, Z = d0 D, s G, c pkS, s M, c Z
    Point base[6], prod[6];
    Fe k[6] = {d0, d0, s, c, s, c};
    base[0] = b, base[1] = d;
    generator(base[2]);
    base[3] = pk;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < 6; ++j) {
        if (j == 4) base[4] = prod[0], base[5] = prod[1];
        signed char digits[kDigits + 1];
        recode_scalar(k[j], digits);
        scalar_mul(prod[j], base[j], digits);
    }
    Point t2, t3;
    add(t2, prod[2], prod[3]);
    add(t3, prod[4], prod[5]);
    sha512::Sha384 h;
    xmd_begin(h);
    i2osp2(h, kElementBytes);
    h.bytes(pk_ser, kElementBytes);
    const Point *framed[4] = {&prod[0], &prod[1], &t2, &t3};
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < 4; ++j) absorb_element(h, *framed[j]);
    h.bytes((const unsigned char *)"Challenge", 9);
    Fe expected;
    hash_to_scalar_finish(expected, h);
    return equal(expected, c);
}

// Finalize after a verified proof: N = r^-1 D for the plain blind r in [1, n - 1], then finalize_hash(input, Ser(N))
P384_HD void unblind_finalize(unsigned char out[kOutputBytes], const Fe &r, const Point &d, const unsigned char *input,
                              long long len) {
    Fe ri;
    inv_mod_n(ri, r);
    signed char digits[kDigits + 1];
    recode_scalar(ri, digits);
    Point u;
    scalar_mul_ct(u, d, digits);
    unsigned char issued[kElementBytes];
    compress(issued, u);
    finalize_hash(out, input, len, issued);
}

#undef P384_CONST
#undef HECUDA_P384_CONSTANTS

}  // namespace p384
}  // namespace hecuda
