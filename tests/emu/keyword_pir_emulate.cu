// CPU replay of the keyword-PIR index maps (csrc/sha256.cuh, csrc/keyword_pir.cuh) and the placement (csrc/cuckoo.hpp):
// the same functions the kernels and hecuda_cuckoo_table_create call, with host SHA-256 supplying the candidates.
// Built with nvcc for the host by tests/test_keyword_pir_emulation.py.
//
//   keyword_pir_emulate sha                          stdin: one hex message per line ("." = empty) -> hex digests
//   keyword_pir_emulate table h evictions size slots multiple fixed expansion load rng seed
//                                                    stdin: "keyword value" hex pairs -> one hex line per bucket
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/cuckoo.hpp"
#include "../../swift-homomorphic-encryption_b200/csrc/keyword_pir.cuh"

using namespace hecuda;

static std::vector<unsigned char> unhex(const std::string &s) {
    std::vector<unsigned char> out;
    if (s == ".") return out;
    for (size_t i = 0; i + 1 < s.size(); i += 2) out.push_back((unsigned char)std::stoi(s.substr(i, 2), nullptr, 16));
    return out;
}

int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode == "sha") {
        std::string line;
        while (std::getline(std::cin, line)) {
            const std::vector<unsigned char> msg = unhex(line);
            unsigned char digest[32];
            sha256::sha256(msg.data(), (long long)msg.size(), digest);
            for (unsigned char b : digest) printf("%02x", b);
            printf(" %llu\n", (unsigned long long)kwpir::keyword_hash(msg.data(), (long long)msg.size()));
        }
        return 0;
    }
    if (mode != "table" || argc != 12) return 2;
    cuckoo::Config c{atoi(argv[2]), atoll(argv[3]), atoll(argv[4]), atoi(argv[5]), atoi(argv[6]) != 0, atoll(argv[7]),
                     atof(argv[8]), atof(argv[9])};
    const cuckoo::Generator rng{atoi(argv[10]), strtoull(argv[11], nullptr, 10)};
    std::vector<unsigned char> keywords, values;
    std::vector<uint64_t> koff{0}, voff{0};
    std::string k, v;
    while (std::cin >> k >> v) {
        const std::vector<unsigned char> kb = unhex(k), vb = unhex(v);
        keywords.insert(keywords.end(), kb.begin(), kb.end());
        values.insert(values.end(), vb.begin(), vb.end());
        koff.push_back(keywords.size());
        voff.push_back(values.size());
    }
    const int64_t count = (int64_t)koff.size() - 1;
    const std::string invalid = cuckoo::validate(c);
    if (!invalid.empty()) {
        printf("error %s\n", invalid.c_str());
        return 0;
    }
    std::vector<uint64_t> hashes((size_t)count);
    for (int64_t i = 0; i < count; ++i) hashes[i] = kwpir::keyword_hash(keywords.data() + koff[i], (long long)(koff[i + 1] - koff[i]));
    std::vector<int64_t> candidates((size_t)count * c.hash_function_count);
    auto candidates_for = [&](int64_t per_table) -> const int64_t * {
        for (int64_t i = 0; i < count; ++i)
            kwpir::hash_indices(hashes[i], per_table, c.hash_function_count, candidates.data() + i * c.hash_function_count);
        return candidates.data();
    };
    cuckoo::Table<decltype(candidates_for)> table(c, count, keywords.data(), koff.data(), hashes.data(), voff.data(), rng,
                                                  candidates_for);
    try {
        table.build();
    } catch (const cuckoo::Failure &f) {
        printf("error %s\n", f.message.c_str());
        return 0;
    }
    // bucket_serialize_kernel's byte map, one bucket per line
    for (const cuckoo::Bucket &b : table.buckets()) {
        long long written = 1;
        printf("%02x", (unsigned)b.slots.size());
        for (int64_t e : b.slots) {
            const long long length = (long long)(voff[e + 1] - voff[e]);
            for (long long j = 0; j < kwpir::slot_size(length); ++j)
                printf("%02x", kwpir::slot_byte(hashes[e], values.data() + voff[e], length, j));
            written += kwpir::slot_size(length);
        }
        if (written != b.size) return 3;  // the size tracked during placement
        printf("\n");
    }
    return 0;
}
