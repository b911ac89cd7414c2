// p384.cuh -- the P-384 field and group (SEC 2, FIPS 186-5) as __host__ __device__ functions, for symmetric_pir.cu's
// OPRF evaluation; tests/emu replays them against oracle/oprf_oracle.py.
//
//   Field   12 x 32-bit little-endian limbs in Montgomery form, R = 2^384.  p = 2^384 - 2^128 - 2^96 + 2^32 - 1 is
//           -1 mod 2^32, so the per-word Montgomery factor -p^-1 mod 2^32 is 1 and each reduction step's multiplier
//           is the low word itself.  Every function returns a value below p.
//   Group   Jacobian coordinates (x = X/Z^2, y = Y/Z^3, the identity has Z = 0), a = -3 doubling (dbl-2001-b) and
//           the general addition (add-2007-bl).
//   Hashing RFC 9380 P384_XMD:SHA-384_SSWU_RO_: expand_message_xmd with SHA-384, hash_to_field (L = 72, count 2),
//           the straight-line simplified SWU of its appendix F.2 with Z = -12 and sqrt_ratio for p = 3 mod 4, and the
//           sum of the two mapped points (cofactor 1).
//   Scalar  k * P for a scalar shared by every thread: the host recodes k once into 96 signed odd 4-bit digits
//           (recode_scalar), so the ladder is a fixed sequence of 4 doublings and one table addition per digit.
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
      0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu)
// p and n are plain integers; kOne .. kGy are in Montgomery form (x R mod p): R, R^2, R^3, b, a = -3, Z = -12,
// sqrt(-Z) = sqrt(12) and the generator; kPMinus2 and kSqrtRatioC1 = (p - 3) / 4 are exponents.

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

// ---------------------------------------------------------------- field
// r = t - p if t (with carry word `top`) >= p, else t
P384_HD void reduce_once(Fe &r, const uint32_t t[kLimbs], uint32_t top) {
    const Fe &p = P384_CONST(kP);
    uint32_t d[kLimbs];
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) {
        const uint64_t s = (uint64_t)t[i] - p.v[i] - borrow;
        d[i] = (uint32_t)s;
        borrow = (s >> 32) & 1;
    }
    const uint32_t keep = (uint32_t)0 - (uint32_t)(borrow & (uint64_t)(top == 0));  // all ones: t < p
    for (int i = 0; i < kLimbs; ++i) r.v[i] = (t[i] & keep) | (d[i] & ~keep);
}

P384_HD void add(Fe &r, const Fe &a, const Fe &b) {
    uint32_t t[kLimbs];
    uint64_t c = 0;
    for (int i = 0; i < kLimbs; ++i) {
        c += (uint64_t)a.v[i] + b.v[i];
        t[i] = (uint32_t)c;
        c >>= 32;
    }
    reduce_once(r, t, (uint32_t)c);
}

P384_HD void sub(Fe &r, const Fe &a, const Fe &b) {
    const Fe &p = P384_CONST(kP);
    uint32_t t[kLimbs];
    uint64_t borrow = 0;
    for (int i = 0; i < kLimbs; ++i) {
        const uint64_t s = (uint64_t)a.v[i] - b.v[i] - borrow;
        t[i] = (uint32_t)s;
        borrow = (s >> 32) & 1;
    }
    const uint32_t mask = (uint32_t)0 - (uint32_t)borrow;  // add p back after a borrow
    uint64_t c = 0;
    for (int i = 0; i < kLimbs; ++i) {
        c += (uint64_t)t[i] + (p.v[i] & mask);
        r.v[i] = (uint32_t)c;
        c >>= 32;
    }
}

P384_HD void neg(Fe &r, const Fe &a) {
    Fe zero = {};
    sub(r, zero, a);
}

// a b R^-1 mod p by CIOS; a may be any value below 2^384 and b below p
P384_HD void mul(Fe &r, const Fe &a, const Fe &b) {
    const Fe &p = P384_CONST(kP);
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
        const uint32_t m = t[0];  // t[0] * (-p^-1 mod 2^32), and -p^-1 = 1
        c = (uint64_t)m * p.v[0] + t[0];
        for (int j = 1; j < kLimbs; ++j) {
            c = (uint64_t)m * p.v[j] + t[j] + (c >> 32);
            t[j - 1] = (uint32_t)c;
        }
        c = (uint64_t)t[kLimbs] + (c >> 32);
        t[kLimbs - 1] = (uint32_t)c;
        t[kLimbs] = t[kLimbs + 1] + (uint32_t)(c >> 32);
    }
    reduce_once(r, t, t[kLimbs]);
}

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

// a^e for a public exponent e (a plain integer), by fixed 4-bit windows
P384_HD void pow_fixed(Fe &r, const Fe &a, const Fe &e) {
    Fe table[16];
    table[0] = P384_CONST(kOne);
    table[1] = a;
    for (int i = 2; i < 16; ++i) mul(table[i], table[i - 1], a);
    r = P384_CONST(kOne);
    for (int w = kDigits - 1; w >= 0; --w) {
        for (int s = 0; s < 4; ++s) sqr(r, r);
        const uint32_t nibble = (e.v[w >> 3] >> (4 * (w & 7))) & 15;
        if (nibble) mul(r, r, table[nibble]);
    }
}

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

// A 72-byte big-endian integer mod p, in Montgomery form: hi 2^384 + lo -> hi R^3 R^-1 + lo R^2 R^-1 = (hi 2^384 + lo) R
P384_HD void from_bytes72(Fe &r, const unsigned char be[72]) {
    Fe hi = {}, lo, a, b;
    for (int i = 0; i < 6; ++i) {
        const unsigned char *q = be + 4 * (5 - i);
        hi.v[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    }
    from_bytes(lo, be + 24);
    mul(a, hi, P384_CONST(kR3));
    mul(b, lo, P384_CONST(kR2));
    add(r, a, b);
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
P384_HD void compress(unsigned char out[kElementBytes], const Point &p) {
    Fe x, y, xp, yp;
    if (!to_affine(x, y, p)) {
        for (int i = 0; i < kElementBytes; ++i) out[i] = 0;
        return;
    }
    from_mont(xp, x);
    from_mont(yp, y);
    out[0] = (unsigned char)(2 | (yp.v[0] & 1));
    to_bytes(out + 1, xp);
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

// expand_message_xmd(msg, DST, 144) with SHA-384 (RFC 9380 5.3.1), DST = HashToGroup-contextString
P384_HD void expand_message_xmd(unsigned char out[144], const unsigned char *msg, long long len) {
    const unsigned char *dst = (const unsigned char *)HECUDA_OPRF_HASH_TO_GROUP_DST;
    sha512::Sha384 s;
    s.init();
    s.zeros(128);  // Z_pad
    s.bytes(msg, len);
    s.byte(0), s.byte(144), s.byte(0);  // I2OSP(len_in_bytes, 2) || I2OSP(0, 1)
    s.bytes(dst, kHashToGroupDstBytes), s.byte(kHashToGroupDstBytes);
    unsigned char b0[48];
    s.finish(b0);
    for (int i = 1; i <= 3; ++i) {
        s.init();
        for (int j = 0; j < 48; ++j) s.byte(i == 1 ? b0[j] : (unsigned char)(b0[j] ^ out[48 * (i - 2) + j]));
        s.byte(i);
        s.bytes(dst, kHashToGroupDstBytes), s.byte(kHashToGroupDstBytes);
        s.finish(out + 48 * (i - 1));
    }
}

// HashToGroup(msg): hash_to_field (two 72-byte field elements), map both, add
P384_HD void hash_to_group(Point &r, const unsigned char *msg, long long len) {
    unsigned char uniform[144];
    expand_message_xmd(uniform, msg, len);
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
P384_HD bool scalar_valid(const Fe &k) {
    if (is_zero(k)) return false;
    const Fe &n = P384_CONST(kN);
    for (int i = kLimbs - 1; i >= 0; --i)
        if (k.v[i] != n.v[i]) return k.v[i] < n.v[i];
    return false;
}

// The recoding of a valid k, done once on the host: k is made odd (k' = n - k and flip = 1 when k is even, since n is
// odd), then k' = sum d_i 16^i with 96 odd digits |d_i| <= 15, d_95 > 0 (regular signed windows).  digits[96] = flip.
P384_HD void recode_scalar(const Fe &k, signed char digits[kDigits + 1]) {
    const Fe &n = P384_CONST(kN);
    Fe w = k;
    const int flip = (k.v[0] & 1) == 0;
    if (flip) {
        uint64_t borrow = 0;
        for (int i = 0; i < kLimbs; ++i) {
            const uint64_t s = (uint64_t)n.v[i] - k.v[i] - borrow;
            w.v[i] = (uint32_t)s;
            borrow = (s >> 32) & 1;
        }
    }
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

P384_HD void generator(Point &g) {
    g.x = P384_CONST(kGx), g.y = P384_CONST(kGy), g.z = P384_CONST(kOne);
}

// RFC 9497 Evaluate's output for one input: SHA-384(I2OSP(len, 2) || input || I2OSP(49, 2) || k HashToGroup(input) ||
// "Finalize"); len < 2^16
P384_HD void oprf_evaluate(unsigned char out[kOutputBytes], const signed char *digits, const unsigned char *input,
                           long long len) {
    Point e, z;
    hash_to_group(e, input, len);
    scalar_mul(z, e, digits);
    unsigned char issued[kElementBytes];
    compress(issued, z);
    sha512::Sha384 s;
    s.init();
    s.byte((uint32_t)(len >> 8)), s.byte((uint32_t)len);
    s.bytes(input, len);
    s.byte(0), s.byte(kElementBytes);
    s.bytes(issued, kElementBytes);
    s.bytes((const unsigned char *)"Finalize", 8);
    s.finish(out);
}

#undef P384_CONST
#undef HECUDA_P384_CONSTANTS

}  // namespace p384
}  // namespace hecuda
