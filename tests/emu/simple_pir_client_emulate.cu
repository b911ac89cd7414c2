// Host replay of the SimplePIR client's arithmetic and index maps (swift-homomorphic-encryption_b200/csrc/
// simple_pir.cuh, process_db.cuh): one command per stdin line, one result line each.
//
//   offsets i j n c k                  -> secret_coefficient(i, j, n) error_coefficient(i, c, k)
//   delta index i cpe epc              -> delta_column
//   extract index i t cpe epc m chunk  -> extract_offset
//   round x p ct                       -> divide_and_round(x, p, 2^ct)
//   results w p planes P_0 Nn_0 ...    -> results_word of the planes' sums
//   integrate r s pt ct                -> integrate
//   bytes bits count c_0 .. c_{count-1} -> coefficientsToBytes as hex
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/simple_pir.cuh"

using namespace hecuda;

static void mu_of(uint64_t p, uint64_t &hi, uint64_t &lo) {
    const spir::spir_u128 mu = ~(spir::spir_u128)0 / p;
    hi = (uint64_t)(mu >> 64), lo = (uint64_t)mu;
}

int main() {
    char cmd[32];
    while (scanf("%31s", cmd) == 1) {
        if (!strcmp(cmd, "offsets")) {
            long long i, j, n, c, k;
            scanf("%lld %lld %lld %lld %lld", &i, &j, &n, &c, &k);
            printf("%lld %lld\n", spir::secret_coefficient(i, j, n), spir::error_coefficient(i, c, k));
        } else if (!strcmp(cmd, "delta")) {
            long long index, i, cpe, epc;
            scanf("%lld %lld %lld %lld", &index, &i, &cpe, &epc);
            printf("%lld\n", spir::delta_column(index, i, cpe, epc));
        } else if (!strcmp(cmd, "extract")) {
            long long index, i, t, cpe, epc, m, chunk;
            scanf("%lld %lld %lld %lld %lld %lld %lld", &index, &i, &t, &cpe, &epc, &m, &chunk);
            printf("%lld\n", spir::extract_offset(index, i, t, cpe, epc, m, chunk));
        } else if (!strcmp(cmd, "round")) {
            unsigned long long x, p;
            int ct;
            scanf("%llu %llu %d", &x, &p, &ct);
            uint64_t hi, lo;
            mu_of(p, hi, lo);
            printf("%llu\n", (unsigned long long)spir::divide_and_round(x, p, hi, lo, ct));
        } else if (!strcmp(cmd, "results")) {
            int w, planes;
            unsigned long long p;
            scanf("%d %llu %d", &w, &p, &planes);
            spir::spir_u128 acc = 0;
            for (int d = 0; d < planes; ++d) {
                unsigned pos, neg;
                scanf("%u %u", &pos, &neg);
                acc = spir::results_add(acc, pos, neg, d, p);
            }
            uint64_t hi, lo;
            mu_of(p, hi, lo);
            printf("%llu\n", (unsigned long long)spir::results_word(acc, w, p, hi, lo));
        } else if (!strcmp(cmd, "integrate")) {
            unsigned long long r, s;
            int pt, ct;
            scanf("%llu %llu %d %d", &r, &s, &pt, &ct);
            printf("%llu\n", (unsigned long long)spir::integrate(r, s, pt, ct));
        } else if (!strcmp(cmd, "bytes")) {
            int bits;
            long long count;
            scanf("%d %lld", &bits, &count);
            std::vector<unsigned long long> c(count);
            for (auto &v : c) scanf("%llu", &v);
            const long long bytes = (count * bits + 7) / 8;
            for (long long b = 0; b < bytes; ++b)
                printf("%02x", procdb::coefficients_byte([&](long long i) { return (uint64_t)c[i]; }, count, bits, b));
            printf("\n");
        } else {
            fprintf(stderr, "unknown command %s\n", cmd);
            return 2;
        }
    }
    return 0;
}
