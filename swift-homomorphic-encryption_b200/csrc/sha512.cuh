// sha512.cuh -- FIPS 180-4 SHA-384 (the SHA-512 compression with the SHA-384 initial value) as __host__ __device__
// functions, for symmetric_pir.cu's hash-to-curve and OPRF Finalize; tests/emu replays them against hashlib.
// `Sha384` is a streaming hasher: absorb bytes in any pieces, then `finish` writes the 48-byte digest.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define SHA5_HD __host__ __device__ __forceinline__
#else
#define SHA5_HD inline
#endif

namespace hecuda {
namespace sha512 {

#define HECUDA_SHA512_K                                                                                                 \
    {0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull, \
     0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull, \
     0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull, \
     0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull, \
     0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull, \
     0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull, \
     0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull, \
     0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull, \
     0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull, \
     0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull, \
     0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull, \
     0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull, \
     0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull, \
     0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull, \
     0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull, \
     0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull}

#ifdef __CUDACC__
static __constant__ uint64_t kRoundDevice[80] = HECUDA_SHA512_K;
#endif
static const uint64_t kRoundHost[80] = HECUDA_SHA512_K;
#undef HECUDA_SHA512_K

SHA5_HD uint64_t round_constant(int i) {
#ifdef __CUDA_ARCH__
    return kRoundDevice[i];
#else
    return kRoundHost[i];
#endif
}

SHA5_HD uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

// One 128-byte block, w[0..15] its big-endian words; w is used as the rolling message schedule.
SHA5_HD void compress(uint64_t h[8], uint64_t w[16]) {
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
#ifdef __CUDA_ARCH__
#pragma unroll 16
#endif
    for (int i = 0; i < 80; ++i) {
        uint64_t wi;
        if (i < 16) {
            wi = w[i];
        } else {
            const uint64_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            const uint64_t s0 = rotr(w15, 1) ^ rotr(w15, 8) ^ (w15 >> 7);
            const uint64_t s1 = rotr(w2, 19) ^ rotr(w2, 61) ^ (w2 >> 6);
            wi = w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
        }
        const uint64_t t1 = k + (rotr(e, 14) ^ rotr(e, 18) ^ rotr(e, 41)) + ((e & f) ^ (~e & g)) + round_constant(i) + wi;
        const uint64_t t2 = (rotr(a, 28) ^ rotr(a, 34) ^ rotr(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
        k = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
    }
    h[0] += a, h[1] += b, h[2] += c, h[3] += d, h[4] += e, h[5] += f, h[6] += g, h[7] += k;
}

// Streaming SHA-384: the block being filled is kept as big-endian words.
struct Sha384 {
    uint64_t h[8];
    uint64_t w[16];
    unsigned long long length;  // bytes absorbed

    SHA5_HD void init() {
        h[0] = 0xcbbb9d5dc1059ed8ull, h[1] = 0x629a292a367cd507ull, h[2] = 0x9159015a3070dd17ull, h[3] = 0x152fecd8f70e5939ull;
        h[4] = 0x67332667ffc00b31ull, h[5] = 0x8eb44a8768581511ull, h[6] = 0xdb0c2e0d64f98fa7ull, h[7] = 0x47b5481dbefa4fa4ull;
        for (int i = 0; i < 16; ++i) w[i] = 0;
        length = 0;
    }
    // byte `length % 128` of the current block; a full block is compressed at once
    SHA5_HD void byte(uint32_t v) {
        const int at = (int)(length & 127);
        w[at >> 3] |= (uint64_t)(v & 0xffu) << (56 - 8 * (at & 7));
        ++length;
        if ((length & 127) == 0) {
            compress(h, w);
            for (int i = 0; i < 16; ++i) w[i] = 0;
        }
    }
    SHA5_HD void bytes(const unsigned char *p, long long n) {
        for (long long i = 0; i < n; ++i) byte(p[i]);
    }
    // `n` zero bytes
    SHA5_HD void zeros(long long n) {
        for (long long i = 0; i < n; ++i) byte(0);
    }
    // 0x80, zeros, then the bit length as a 128-bit big-endian integer (its high word is 0 below 2^61 bytes)
    SHA5_HD void finish(unsigned char out[48]) {
        const unsigned long long bits = length * 8ull;
        byte(0x80);
        while ((length & 127) != 112) byte(0);
        for (int i = 0; i < 8; ++i) byte(0);
        for (int i = 7; i >= 0; --i) byte((uint32_t)(bits >> (8 * i)));
        for (int i = 0; i < 48; ++i) out[i] = (unsigned char)(h[i >> 3] >> (56 - 8 * (i & 7)));
    }
};

SHA5_HD void sha384(const unsigned char *msg, long long len, unsigned char out[48]) {
    Sha384 s;
    s.init();
    s.bytes(msg, len);
    s.finish(out);
}

}  // namespace sha512
}  // namespace hecuda
