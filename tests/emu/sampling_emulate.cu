// sampling_emulate.cu -- replays on the host the __host__ __device__ sampling maps the client kernels call
// (csrc/sampling.cuh) over the CTR_DRBG segment chain of csrc/drbg.cuh.  Prints coefficients first .. first + count - 1
// of one seed's stream, space-separated: ternary values in {0, 1, 2} (before the reference's "- 1"), or CBD values.
//   usage: sampling_emulate <seed hex (64 chars)> ternary <first> <count>
//          sampling_emulate <seed hex (64 chars)> cbd <sigma> <first> <count>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/sampling.cuh"

using namespace hecuda;
using namespace hecuda::drbg;

int main(int argc, char **argv) {
    if (argc < 5 || std::strlen(argv[1]) != 64) return 2;
    const bool ternary = std::strcmp(argv[2], "ternary") == 0;
    if (!ternary && argc < 6) return 2;
    unsigned char seed[32], sbox[256];
    u32w te0[256];
    for (int i = 0; i < 32; ++i) {
        unsigned v = 0;
        std::sscanf(argv[1] + 2 * i, "%2x", &v);
        seed[i] = (unsigned char)v;
    }
    int words = 0;
    u64 mask = 0;
    if (!ternary && !cbd_shape(std::atof(argv[3]), words, mask)) return 3;
    const long long first = std::atoll(argv[ternary ? 3 : 4]), count = std::atoll(argv[ternary ? 4 : 5]);
    const long long bytes = (first + count) * (ternary ? kTernaryBytes : 8LL * words);
    const int segments = (int)((bytes + kSegmentBytes - 1) / kSegmentBytes);
    make_tables(sbox, te0);
    // the chain drbg_chain_kernel walks: (round keys, V) of every segment
    std::vector<u32w> rks((size_t)segments * kRoundKeyWords);
    std::vector<u64> ctrs((size_t)segments * 2);
    u32w key[4] = {0, 0, 0, 0}, rk[kRoundKeyWords], provided[8], b0[4], b1[4];
    for (int i = 0; i < 8; ++i)
        provided[i] = ((u32w)seed[4 * i] << 24) | ((u32w)seed[4 * i + 1] << 16) | ((u32w)seed[4 * i + 2] << 8) | seed[4 * i + 3];
    u64 hi = 0, lo = 0;
    for (int s = -1; s < segments; ++s) {
        expand_key(key, rk, sbox);
        if (s >= 0) {
            std::memcpy(&rks[(size_t)s * kRoundKeyWords], rk, sizeof(rk));
            ctrs[2 * s] = hi;
            ctrs[2 * s + 1] = lo;
            const u64 l = lo + kSegmentBlocks;
            hi += l < lo ? 1 : 0;
            lo = l;
        }
        counter_block(hi, lo, 1, b0);
        counter_block(hi, lo, 2, b1);
        encrypt_block(b0, rk, te0, sbox);
        encrypt_block(b1, rk, te0, sbox);
        drbg_absorb(key, hi, lo, b0, b1, s < 0 ? provided : nullptr);
    }
    StreamReader st;
    st.rk = rks.data();
    st.ctr = ctrs.data();
    st.sbox = sbox;
    st.te0 = te0;
    for (long long j = first; j < first + count; ++j) {
        if (ternary)
            std::printf("%llu ", (unsigned long long)ternary_value(st, j));
        else
            std::printf("%d ", cbd_value(st, j, words, mask));
    }
    std::printf("\n");
    return 0;
}
