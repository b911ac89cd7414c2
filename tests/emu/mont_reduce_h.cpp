// Host check of mont_reduce_h against mont_reduce (csrc/modarith.cuh).  Reads lines "p acc_hi acc_lo" (decimal) and
// prints "mont_reduce mont_reduce_h" for each, with ninv = -p^-1 mod 2^64 computed as context.cu does.
#include <cstdio>

#include "../../swift-homomorphic-encryption_b200/csrc/modarith.cuh"

using namespace hecuda;

int main() {
    unsigned long long p, hi, lo;
    while (std::scanf("%llu %llu %llu", &p, &hi, &lo) == 3) {
        u64 inv = p;
        for (int i = 0; i < 6; ++i) inv *= 2 - p * inv;
        const u128 acc = ((u128)hi << 64) | lo;
        std::printf("%llu %llu\n", (unsigned long long)mont_reduce(acc, p, 0 - inv), (unsigned long long)mont_reduce_h(acc, p));
    }
    return 0;
}
