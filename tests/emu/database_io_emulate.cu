// Host replay of saving and loading processed PIR databases: the tag walk, the chunk planner and the tag offsets of
// swift-homomorphic-encryption_b200/csrc/database_io.hpp, and the per-plaintext offset map (tagged_rows_offset) and bit
// codec (codec_unpack, codec_pack) that the load and serialize kernels of codec.cu call, evaluated on the CPU chunk by
// chunk as the device pipelines stage them.
//
//   load N budget L q_0 .. q_{L-1}     stdin: the file as hex
//        -> "walk <error> <value> <at> <count>", then "tags t_0 .. t_count", then one "chunk first count" per chunk, then
//           per plaintext "present r_0 .. r_{L*N-1}" (the resident words), then "bad <index or -1>"
//   save N budget L q_0 .. q_{L-1}     stdin: count, then per plaintext: present flag and L*N residues
//        -> "tags ...", "chunk ..." lines, then the file as hex, once from the byte kernel and once from the 8-byte kernel
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/database_io.hpp"
#include "../../swift-homomorphic-encryption_b200/csrc/kernels.cuh"

using namespace hecuda;

struct Shape {
    int n = 0, rows = 0;
    std::vector<int> width;
    std::vector<long long> byte_offset{0};
    std::vector<u64> modulus;
    long long budget = 0;
};

static int ceil_log2(u64 q) {
    int bits = 0;
    while (bits < 64 && (q - 1) >> bits) ++bits;
    return bits;
}

static bool parse_shape(int argc, char **argv, Shape &s) {
    if (argc < 5) return false;
    s.n = atoi(argv[2]);
    s.budget = atoll(argv[3]);
    s.rows = atoi(argv[4]);
    if (argc < 5 + s.rows) return false;
    for (int r = 0; r < s.rows; ++r) {
        s.modulus.push_back(strtoull(argv[5 + r], nullptr, 10));
        s.width.push_back(ceil_log2(s.modulus.back()));
        s.byte_offset.push_back(s.byte_offset.back() + ((long long)s.n * s.width.back() + 7) / 8);
    }
    return true;
}

static void print_plan(const std::vector<long long> &tag, long long count, long long budget, std::vector<dbio::Chunk> &plan) {
    printf("tags");
    for (long long t : tag) printf(" %lld", t);
    printf("\n");
    plan = dbio::plan_chunks(tag, 0, count, budget);
    for (const dbio::Chunk &ch : plan) printf("chunk %lld %lld\n", ch.first, ch.count);
}

static int run_load(const Shape &s) {
    std::string hex;
    std::cin >> hex;
    if (hex == ".") hex.clear();
    std::vector<unsigned char> file;
    for (size_t k = 0; k + 1 < hex.size(); k += 2) file.push_back((unsigned char)strtoul(hex.substr(k, 2).c_str(), nullptr, 16));
    std::vector<long long> tag;
    const long long plaintext_bytes = s.byte_offset.back();
    const dbio::TagWalk w = dbio::walk_tags(file.data(), (long long)file.size(), plaintext_bytes, tag);
    printf("walk %d %u %lld %lld\n", (int)w.error, w.value, w.at, w.count);
    if (w.error != dbio::TagWalk::kOk) return 0;
    std::vector<dbio::Chunk> plan;
    print_plan(tag, w.count, s.budget, plan);
    std::vector<u64> rows((size_t)(w.count * s.rows * s.n));
    std::vector<int> present((size_t)w.count);
    unsigned long long bad = ~0ull;
    for (const dbio::Chunk &ch : plan) {
        const long long base = tag[(size_t)ch.first];
        // the staging buffer holds exactly the chunk's bytes
        const std::vector<unsigned char> staged(file.begin() + base, file.begin() + tag[(size_t)(ch.first + ch.count)]);
        for (long long poly = 0; poly < ch.count; ++poly) {
            const long long offset = tagged_rows_offset(tag.data() + ch.first, base, poly);  // poly_load_kernel
            present[(size_t)(ch.first + poly)] = offset >= 0;
            if (offset < 0) continue;
            for (int row = 0; row < s.rows; ++row)
                for (int i = 0; i < s.n; ++i) {
                    const long long row_bytes = s.byte_offset[row + 1] - s.byte_offset[row];
                    const u64 v = codec_unpack(staged.data() + offset + s.byte_offset[row], row_bytes, s.width[row], i);
                    if (v >= s.modulus[row]) bad = std::min(bad, (unsigned long long)(ch.first + poly) * s.rows + row);
                    rows[(size_t)(((ch.first + poly) * s.rows + row) * s.n + i)] = v;
                }
        }
    }
    for (long long p = 0; p < w.count; ++p) {
        std::string line = std::to_string(present[(size_t)p]);
        for (long long k = 0; k < (long long)s.rows * s.n; ++k) line += " " + std::to_string(rows[(size_t)(p * s.rows * s.n + k)]);
        puts(line.c_str());
    }
    printf("bad %lld\n", bad == ~0ull ? -1ll : (long long)bad);
    return 0;
}

static std::string to_hex(const std::vector<unsigned char> &bytes) {
    static const char *digits = "0123456789abcdef";
    std::string out;
    for (unsigned char b : bytes) out += std::string(1, digits[b >> 4]) + digits[b & 15];
    return out;
}

static int run_save(const Shape &s) {
    long long count = 0;
    if (!(std::cin >> count)) return 3;
    std::vector<unsigned char> present((size_t)count);
    std::vector<u64> rows((size_t)(count * s.rows * s.n));
    for (long long p = 0; p < count; ++p) {
        int flag = 0;
        if (!(std::cin >> flag)) return 3;
        present[(size_t)p] = (unsigned char)flag;
        for (long long k = 0; k < (long long)s.rows * s.n; ++k)
            if (!(std::cin >> rows[(size_t)(p * s.rows * s.n + k)])) return 3;
    }
    std::vector<long long> tag;
    dbio::tag_offsets(present.data(), count, s.byte_offset.back(), tag);
    std::vector<dbio::Chunk> plan;
    print_plan(tag, count, s.budget, plan);
    for (int words = 0; words < 2; ++words) {
        std::vector<unsigned char> file((size_t)tag.back(), 0xee);  // every byte must be written
        file[0] = dbio::kVersion;
        for (int k = 0; k < 4; ++k) file[(size_t)(1 + k)] = (unsigned char)(count >> (8 * k));
        for (const dbio::Chunk &ch : plan) {
            const long long base = tag[(size_t)ch.first];
            std::vector<unsigned char> staged((size_t)(tag[(size_t)(ch.first + ch.count)] - base), 0xee);
            for (long long poly = 0; poly < ch.count; ++poly) {
                const long long offset = tagged_rows_offset(tag.data() + ch.first, base, poly);
                staged[(size_t)(tag[(size_t)(ch.first + poly)] - base)] = offset >= 0;  // write_tag
                if (offset < 0) continue;
                for (int row = 0; row < s.rows; ++row) {
                    const u64 *src = rows.data() + ((ch.first + poly) * s.rows + row) * s.n;
                    const long long row_bytes = s.byte_offset[row + 1] - s.byte_offset[row];
                    unsigned char *dst = staged.data() + offset + s.byte_offset[row];
                    if (words) {  // poly_serialize_words_kernel: 64 stream bits a thread, most significant byte first
                        for (long long j = 0; j < row_bytes / 8; ++j) {
                            const u64 value = codec_pack(src, s.n, s.width[row], 0, 64 * j, 64);
                            for (int k = 0; k < 8; ++k) dst[8 * j + k] = (unsigned char)(value >> (56 - 8 * k));
                        }
                    } else {  // poly_serialize_kernel: one byte a thread
                        for (long long j = 0; j < row_bytes; ++j) dst[j] = (unsigned char)codec_pack(src, s.n, s.width[row], 0, 8 * j, 8);
                    }
                }
            }
            memcpy(file.data() + base, staged.data(), staged.size());
        }
        puts(to_hex(file).c_str());
    }
    return 0;
}

int main(int argc, char **argv) {
    Shape s;
    if (argc < 2 || !parse_shape(argc, argv, s)) return 2;
    if (!strcmp(argv[1], "load")) return run_load(s);
    if (!strcmp(argv[1], "save")) return run_save(s);
    return 2;
}
