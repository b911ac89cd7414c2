// Host replay of the SimplePIR response arithmetic (swift-homomorphic-encryption_b200/csrc/simple_pir.cuh): the digit
// split, the s32 slice sums, their widening and the final mask, in the order response_kernel applies them.
//
//   response pt ct k      stdin: k DB' values, then k request words (decimal)
//        -> one line: the response word, then the largest slice sum seen (which must stay below 2^31)
//   layout rows cols      -> the a_offset of every (r, c) then the b_offset of every (q = r, c), one per line
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/simple_pir.cuh"

using namespace hecuda::spir;

int main(int argc, char **argv) {
    if (argc >= 5 && !strcmp(argv[1], "response")) {
        const int pt = atoi(argv[2]), ct = atoi(argv[3]);
        const long long k = atoll(argv[4]);
        std::vector<unsigned long long> db(k), req(k);
        for (auto &v : db) scanf("%llu", &v);
        for (auto &v : req) scanf("%llu", &v);
        uint64_t acc = 0;
        long long largest = 0;
        for (long long s0 = 0; s0 < k; s0 += kSliceColumns)
            for (int i = 0; i < digits(pt); ++i)
                for (int j = 0; j < digits(ct); ++j) {
                    if (!pair_live(i, j, ct)) continue;
                    long long sum = 0;  // what the s32 MMA accumulator holds: checked against 2^31 below
                    for (long long c = s0; c < k && c < s0 + kSliceColumns; ++c)
                        sum += (long long)db_digit(db[c], i) * query_digit(req[c], ct, j);
                    if (sum > largest) largest = sum;
                    acc = widen(acc, (uint32_t)sum, i, j);
                }
        printf("%llu %lld\n", (unsigned long long)finish(acc, ct), largest);
        return 0;
    }
    if (argc >= 4 && !strcmp(argv[1], "layout")) {
        const long long rows = atoll(argv[2]), cols = atoll(argv[3]), tiles = cols / kTileCols;
        for (long long r = 0; r < rows; ++r)
            for (long long c = 0; c < cols; ++c) printf("%lld\n", a_offset(r, c, tiles));
        for (long long r = 0; r < rows; ++r)
            for (long long c = 0; c < cols; ++c) printf("%lld\n", b_offset(r, c, tiles));
        return 0;
    }
    fprintf(stderr, "usage: response pt ct k | layout rows cols\n");
    return 2;
}
