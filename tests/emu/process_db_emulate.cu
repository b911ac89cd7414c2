// Host replay of the database-processing index maps (swift-homomorphic-encryption_b200/csrc/process_db.cuh): the
// same __host__ __device__ functions the packing and gather kernels call, evaluated on the CPU.
//
//   pir  N t entry_size encode dim_count dim0 [dim1] entry_count with_offsets   stdin: one hex entry per line ("." = empty)
//        -> one line per plaintext: present c_0 .. c_{N-1}            (what pir_pack_kernel writes)
//   pnns logN rows cols baby giant t reduce resident                 stdin: rows * cols signed values
//        -> first line "bad 0|1", then one line per plaintext: the SIMD slot values 0 .. N-1 before encodeSimd's
//           scatter and inverse NTT (what pnns_gather_kernel writes at Eval position matrix[slot])
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/process_db.cuh"

using namespace hecuda::procdb;

static int run_pir(int argc, char **argv) {
    if (argc < 9) return 2;
    const long long n = atoll(argv[2]);
    const uint64_t t = strtoull(argv[3], nullptr, 10);
    const long long entry_size = atoll(argv[4]);
    const bool encode = atoi(argv[5]) != 0;
    const int dim_count = atoi(argv[6]);
    const long long dim0 = atoll(argv[7]), dim1 = dim_count == 2 ? atoll(argv[8]) : 1;
    const int at = dim_count == 2 ? 9 : 8;
    if (argc < at + 2) return 2;
    const long long entry_count = atoll(argv[at]);
    const bool with_offsets = atoi(argv[at + 1]) != 0;
    std::vector<unsigned char> bytes;
    std::vector<uint64_t> offsets{0};
    std::string line;
    for (long long i = 0; i < entry_count; ++i) {
        if (!(std::cin >> line)) return 3;
        if (line != ".")
            for (size_t k = 0; k + 1 < line.size(); k += 2) bytes.push_back((unsigned char)strtoul(line.substr(k, 2).c_str(), nullptr, 16));
        offsets.push_back(bytes.size());
    }
    PirShape s = pir_shape(n, t, entry_count, entry_size, encode, dim0 * dim1, dim0);
    s.entries = bytes.data();
    s.offsets = with_offsets ? offsets.data() : nullptr;
    const long long count = pir_chunk_count(s) * s.per_chunk;
    std::string out;
    for (long long index = 0; index < count; ++index) {
        const PirPiece p = pir_piece(s, index);
        std::vector<uint64_t> row(n);
        bool any = false;
        for (long long i = 0; i < n; ++i) any |= (row[i] = pir_coefficient(s, p, i)) != 0;
        out += any ? "1" : "0";
        for (long long i = 0; i < n; ++i) out += " " + std::to_string(row[i]);
        out += "\n";
    }
    fputs(out.c_str(), stdout);
    return 0;
}

static int run_pnns(int argc, char **argv) {
    if (argc < 10) return 2;
    PnnsShape s{};
    s.logn = atoi(argv[2]);
    s.rows = atoll(argv[3]);
    s.cols = atoll(argv[4]);
    s.baby = atoi(argv[5]);
    s.giant = atoi(argv[6]);
    const uint64_t t = strtoull(argv[7], nullptr, 10);
    const bool reduce = atoi(argv[8]) != 0, resident = atoi(argv[9]) != 0;
    const int n = 1 << s.logn;
    s.results = (s.rows + n - 1) / n;
    s.dimension = 1;
    while (s.dimension < s.cols) s.dimension <<= 1;
    std::vector<long long> values((size_t)(s.rows * s.cols));
    for (auto &v : values)
        if (!(std::cin >> v)) return 3;
    const long long count = resident ? s.results * s.giant * s.baby : (long long)s.dimension * s.results;
    bool bad = false;
    std::string out;
    for (long long item = 0; item < count; ++item) {
        int d;
        long long r;
        bool live = true;
        if (resident)
            live = pnns_resident(s, item, d, r);
        else
            pnns_plaintext(s, item, d, r);
        for (int slot = 0; slot < n; ++slot) {
            uint64_t v = 0;
            if (live) {
                const long long e = pnns_element(s, d, r, slot);
                if (e >= 0) v = pnns_signed_value(values[(size_t)e], t, reduce, bad);
            }
            out += (slot ? " " : "") + std::to_string(v);
        }
        out += "\n";
    }
    printf("bad %d\n", bad ? 1 : 0);
    fputs(out.c_str(), stdout);
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    if (!strcmp(argv[1], "pir")) return run_pir(argc, argv);
    if (!strcmp(argv[1], "pnns")) return run_pnns(argc, argv);
    return 2;
}
