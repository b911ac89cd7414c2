// Host build of the PNNS client helpers of csrc/process_db.cuh (the float front end, the .denseRow and .denseColumn
// maps and the plaintext CRT), so tests/test_pnns_client_emulation.py can check exactly what the kernels compute.
// Compiled with -Xcompiler -ffp-contract=off.  Reads its inputs from stdin:
//   norm S ROWS COLS  then ROWS x COLS float bit patterns (hex)   -> per value: the Int64, or "bad"
//   dense_row ROWS COLS LOGN                                      -> per plaintext, per slot: the value index or -1
//   dense_column ROWS COLS LOGN                                   -> per row-major element: plaintext and slot
//   crt K T_0 .. T_{K-1} S COUNT  then COUNT x K residues          -> per value: the centred integer and the float bits
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/process_db.cuh"

using namespace hecuda::procdb;

static uint64_t inv_mod(uint64_t a, uint64_t m) {
    __int128 r0 = m, r1 = a % m, s0 = 0, s1 = 1;
    while (r1) {
        const __int128 q = r0 / r1, r = r0 - q * r1, s = s0 - q * s1;
        r0 = r1, r1 = r, s0 = s1, s1 = s;
    }
    return (uint64_t)(s0 < 0 ? s0 + m : s0);
}

int main() {
    char mode[32];
    if (scanf("%31s", mode) != 1) return 2;
    if (!strcmp(mode, "norm")) {
        long long s, rows, cols;
        if (scanf("%lld %lld %lld", &s, &rows, &cols) != 3) return 2;
        std::vector<float> v((size_t)(rows * cols));
        for (auto &x : v) {
            unsigned bits;
            if (scanf("%x", &bits) != 1) return 2;
            memcpy(&x, &bits, 4);
        }
        for (long long r = 0; r < rows; ++r) {
            const float norm = pnns_row_norm(&v[(size_t)(r * cols)], cols);
            for (long long c = 0; c < cols; ++c) {
                bool bad = false;
                const long long x = pnns_scaled_value(v[(size_t)(r * cols + c)], (float)s, norm, bad);
                if (bad) printf("bad\n");
                else printf("%lld\n", x);
            }
        }
    } else if (!strcmp(mode, "dense_row")) {
        long long rows, cols;
        int logn;
        if (scanf("%lld %lld %d", &rows, &cols, &logn) != 3) return 2;
        const long long count = pnns_dense_row_count(rows, cols, logn);
        for (long long p = 0; p < count; ++p)
            for (long long slot = 0; slot < (1ll << logn); ++slot) printf("%lld\n", pnns_dense_row_element(rows, cols, logn, p, slot));
    } else if (!strcmp(mode, "dense_column")) {
        long long rows, cols;
        int logn;
        if (scanf("%lld %lld %d", &rows, &cols, &logn) != 3) return 2;
        printf("%lld\n", pnns_dense_column_count(rows, cols, logn));
        for (long long r = 0; r < rows; ++r)
            for (long long c = 0; c < cols; ++c) {
                long long p, slot;
                pnns_dense_column_slot(rows, cols, logn, r, c, p, slot);
                printf("%lld %lld\n", p, slot);
            }
    } else if (!strcmp(mode, "crt")) {
        PnnsCrt crt{};
        if (scanf("%d", &crt.count) != 1 || crt.count < 1 || crt.count > 8) return 2;
        crt.product = 1;
        for (int i = 0; i < crt.count; ++i) {
            if (scanf("%llu", (unsigned long long *)&crt.t[i]) != 1) return 2;
            crt.product *= crt.t[i];
        }
        for (int i = 0; i < crt.count; ++i) {
            crt.punct[i] = crt.product / crt.t[i];
            crt.inv[i] = inv_mod(crt.punct[i] % crt.t[i], crt.t[i]);
        }
        long long s, count;
        if (scanf("%lld %lld", &s, &count) != 2) return 2;
        for (long long j = 0; j < count; ++j) {
            uint64_t x[8];
            for (int i = 0; i < crt.count; ++i)
                if (scanf("%llu", (unsigned long long *)&x[i]) != 1) return 2;
            const long long v = pnns_crt_signed(crt, x);
            const float d = pnns_distance(v, s);
            unsigned bits;
            memcpy(&bits, &d, 4);
            printf("%lld %08x\n", v, bits);
        }
    } else {
        return 2;
    }
    return 0;
}
