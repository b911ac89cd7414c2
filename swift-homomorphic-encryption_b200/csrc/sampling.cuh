// sampling.cuh -- the reference's maps from a NistAes128Ctr byte stream to secret-key and error coefficients, as
// __host__ __device__ functions shared by client.cu and its host-side emulation test (tests/emu/sampling_emulate.cu).
//
//   PolyRq.randomizeTernary(using:)                        PolyRq/PolyRq+Randomize.swift:87-104
//   PolyRq.randomizeCenteredBinomialDistribution(...)      PolyRq/PolyRq+Randomize.swift:120-160
//   rng.next() -> T: sizeof(T) stream bytes, little-endian Random/PseudoRandomNumberGenerator.swift:37-43
//
// A seed's stream is the chain of 4096-byte segments drbg.cu walks (drbg_chains): segment s is AES-128-CTR under round
// keys rk[s] from counter V_s + 1.  Coefficient j of either map reads a fixed number of bytes at offset j * bytes, so a
// thread finds its coefficient's bytes directly; they may straddle two segments (12-byte ternary coefficients do).
#pragma once
#include "drbg.cuh"

namespace hecuda {
namespace drbg {

constexpr int kTernaryBytes = 12;  // one UInt64, then one UInt32
constexpr int kMaxCbdWords = 32;   // 64-bit trial words per CBD coefficient (k <= 1024)

// The stream of one seed: `rk` (segments x kRoundKeyWords) and `ctr` (segments x 2: V_s as hi, lo) of its chain.
// Keeps the last block it encrypted, so consecutive reads from one block cost one encryption.
struct StreamReader {
    const u32w *rk;
    const u64 *ctr;
    const unsigned char *sbox;
    const u32w *te0;
    long long cached = -1;
    u32w blk[4];

    HE_HD u32w le32(u32w w) { return (w >> 24) | ((w >> 8) & 0xff00u) | ((w << 8) & 0xff0000u) | (w << 24); }
    // the little-endian UInt32 at byte offset p (a multiple of 4) of the stream
    HE_HD u32w word32(long long p) {
        const long long g = p >> 4;
        if (g != cached) {
            const long long s = g / kSegmentBlocks;
            counter_block(ctr[2 * s], ctr[2 * s + 1], 1 + (u64)(g - s * kSegmentBlocks), blk);
            encrypt_block(blk, rk + s * kRoundKeyWords, te0, sbox);
            cached = g;
        }
        return le32(blk[(p >> 2) & 3]);
    }
    HE_HD u64 word64(long long p) { return (u64)word32(p) | ((u64)word32(p + 4) << 32); }
};

// randomizeTernary: (UInt64 << 32 | UInt32) mod 3 of coefficient j; the coefficient is this minus 1 modulo each q_i
HE_HD u64 ternary_value(StreamReader &st, long long j) {
    const long long p = j * kTernaryBytes;
    const u64 hi = st.word64(p);
    const u64 lo = st.word32(p + 8);
    return (u64)((((u128)hi << 32) | lo) % 3);
}

// The CBD shape of a standard deviation: k = ceil(2 sigma^2) trials per side, 2 ceil(k / 64) words per coefficient,
// the last word of each half masked to k mod 64 bits (no mask when 64 divides k).  Returns false past kMaxCbdWords.
inline bool cbd_shape(double sigma, int &words, u64 &mask) {
    const double k_real = 2.0 * sigma * sigma;
    long long k = (long long)k_real;
    if ((double)k < k_real) ++k;
    words = (int)(2 * ((k + 63) / 64));
    mask = (k % 64) ? (((u64)1 << (k % 64)) - 1) : ~(u64)0;
    return k >= 1 && words <= kMaxCbdWords;
}

// randomizeCenteredBinomialDistribution: popcount(positive half) - popcount(negative half) of coefficient j
HE_HD int cbd_value(StreamReader &st, long long j, int words, u64 mask) {
    const long long p = j * 8LL * words;
    const int half = words >> 1;
    int pos = 0, neg = 0;
    for (int w = 0; w < words; ++w) {
        u64 x = st.word64(p + 8LL * w);
        if (w == half - 1 || w == words - 1) x &= mask;
#if defined(__CUDA_ARCH__)
        const int bits = __popcll(x);
#else
        const int bits = __builtin_popcountll(x);
#endif
        if (w < half)
            pos += bits;
        else
            neg += bits;
    }
    return pos - neg;
}

// a small signed value as a residue modulo p (subtractMod / the negation of a CBD count)
HE_HD u64 signed_residue(long long v, u64 p) { return v >= 0 ? (u64)v : p - (u64)(-v); }

}  // namespace drbg
}  // namespace hecuda
