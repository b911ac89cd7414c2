// Host check of wide_to_double (csrc/hostmath.hpp), the rounding of the noise budget's infinity norm.  Reads lines
// "w x_0 .. x_{w-1}" (decimal words, little-endian) and prints the IEEE-754 bits of the double for each, in decimal.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/hostmath.hpp"

using hecuda::host::u64;

int main() {
    int w;
    while (std::scanf("%d", &w) == 1) {
        std::vector<u64> x(w > 0 ? w : 1);
        for (int i = 0; i < w; ++i)
            if (std::scanf("%llu", &x[i]) != 1) return 1;
        const double d = hecuda::host::wide_to_double(x.data(), w);
        u64 bits;
        std::memcpy(&bits, &d, sizeof bits);
        std::printf("%llu\n", bits);
    }
    return 0;
}
