// sha256.cuh -- FIPS 180-4 SHA-256 as __host__ __device__ functions (keyword_pir.cu's hashes; tests/emu replays them
// against hashlib).  Two entry points: `sha256` for a message of any length, and `first8_9` for the 9-byte
// message of HashKeyword.indexFromHash (HashBucket.swift:244-257), which fits one block and is padded in registers.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define SHA_HD __host__ __device__ __forceinline__
#else
#define SHA_HD inline
#endif

namespace hecuda {
namespace sha256 {

#define HECUDA_SHA256_K                                                                                                \
    {0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,           \
     0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,           \
     0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,           \
     0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,           \
     0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,           \
     0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,           \
     0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,           \
     0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u}

#ifdef __CUDACC__
static __constant__ uint32_t kRoundDevice[64] = HECUDA_SHA256_K;
#endif
static const uint32_t kRoundHost[64] = HECUDA_SHA256_K;
#undef HECUDA_SHA256_K

SHA_HD uint32_t round_constant(int i) {
#ifdef __CUDA_ARCH__
    return kRoundDevice[i];
#else
    return kRoundHost[i];
#endif
}

SHA_HD uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
SHA_HD uint32_t bswap(uint32_t x) {
    return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
}

SHA_HD void init(uint32_t h[8]) {
    h[0] = 0x6a09e667u, h[1] = 0xbb67ae85u, h[2] = 0x3c6ef372u, h[3] = 0xa54ff53au;
    h[4] = 0x510e527fu, h[5] = 0x9b05688cu, h[6] = 0x1f83d9abu, h[7] = 0x5be0cd19u;
}

// One 64-byte block, w[0..15] its big-endian words; w is used as the rolling message schedule.
SHA_HD void compress(uint32_t h[8], uint32_t w[16]) {
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 64; ++i) {
        uint32_t wi;
        if (i < 16) {
            wi = w[i];
        } else {
            const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            const uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
            const uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
            wi = w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
        }
        const uint32_t t1 = k + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + round_constant(i) + wi;
        const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        k = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
    }
    h[0] += a, h[1] += b, h[2] += c, h[3] += d, h[4] += e, h[5] += f, h[6] += g, h[7] += k;
}

// Byte p of the padded message: the message, 0x80, zeros, then the bit length as a big-endian UInt64.
SHA_HD uint32_t padded_byte(const unsigned char *msg, long long len, long long total, long long p) {
    if (p < len) return msg[p];
    if (p == len) return 0x80u;
    if (p >= total - 8) return (uint32_t)(((unsigned long long)len * 8ull >> (8 * (total - 1 - p))) & 0xffu);
    return 0u;
}

// SHA-256 of `len` bytes -> the state words h[0..7] (the digest is their big-endian bytes).
SHA_HD void digest_words(const unsigned char *msg, long long len, uint32_t h[8]) {
    init(h);
    const long long total = ((len + 8) / 64 + 1) * 64;
    for (long long block = 0; block < total; block += 64) {
        uint32_t w[16];
        if (block + 64 <= len) {  // a whole block of message bytes
            for (int i = 0; i < 16; ++i) {
                const unsigned char *p = msg + block + 4 * i;
                w[i] = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
            }
        } else {
            for (int i = 0; i < 16; ++i) {
                uint32_t v = 0;
                for (int j = 0; j < 4; ++j) v = (v << 8) | padded_byte(msg, len, total, block + 4 * i + j);
                w[i] = v;
            }
        }
        compress(h, w);
    }
}

SHA_HD void sha256(const unsigned char *msg, long long len, unsigned char out[32]) {
    uint32_t h[8];
    digest_words(msg, len, h);
    for (int i = 0; i < 32; ++i) out[i] = (unsigned char)(h[i >> 2] >> (24 - 8 * (i & 3)));
}

// The first 8 digest bytes read as a little-endian UInt64 (HashKeyword.hash, HashBucket.swift:264-269).
SHA_HD uint64_t first8_le(const uint32_t h[8]) { return (uint64_t)bswap(h[0]) | ((uint64_t)bswap(h[1]) << 32); }

SHA_HD uint64_t first8(const unsigned char *msg, long long len) {
    uint32_t h[8];
    digest_words(msg, len, h);
    return first8_le(h);
}

// first8(bigEndian(value) || byte): one block, 72 message bits.
SHA_HD uint64_t first8_9(uint64_t value, uint32_t byte) {
    uint32_t h[8], w[16];
    init(h);
    w[0] = (uint32_t)(value >> 32);
    w[1] = (uint32_t)value;
    w[2] = ((byte & 0xffu) << 24) | 0x800000u;
    for (int i = 3; i < 15; ++i) w[i] = 0;
    w[15] = 72;
    compress(h, w);
    return first8_le(h);
}

}  // namespace sha256
}  // namespace hecuda
