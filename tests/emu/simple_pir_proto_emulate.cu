// simple_pir_proto_emulate.cu -- runs the library's SimplePIRRequest walk (simple_pir_proto.hpp) and the device decode
// and encode maps (simple_pir.cuh) on the CPU, visiting the virtual byte stream as proto_decode_kernel does.
//
//   decode <columns> <row_base> <col_tiles> <ct> <word32>   stdin: a SimplePIRRequest as hex
//       -> "error <code> <what>" on a walk refusal, else "flags <f>" (f: the ProtoFlag bits the kernels would set,
//          the count check included) then "<b_offset> <value mod 2^ct>" per decoded varint with index < row x col
//   encode <rows> <columns> <ct> <acc ...>   -> the SimplePIRResponse as hex ("." when empty), then its capacity
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/simple_pir.cuh"
#include "../../swift-homomorphic-encryption_b200/csrc/simple_pir_proto.hpp"

using namespace hecuda;

static std::vector<unsigned char> read_hex() {
    std::string s;
    std::cin >> s;
    std::vector<unsigned char> b;
    if (s == ".") return b;
    for (size_t i = 0; i + 1 < s.size(); i += 2) b.push_back((unsigned char)std::stoi(s.substr(i, 2), nullptr, 16));
    return b;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const std::string cmd = argv[1];
    if (cmd == "decode" && argc == 7) {
        const long long columns = atoll(argv[2]), row_base = atoll(argv[3]), col_tiles = atoll(argv[4]);
        const int ct = atoi(argv[5]);
        const bool word32 = atoi(argv[6]) != 0;
        const std::vector<unsigned char> b = read_hex();
        proto::Error e;
        spirproto::Request r;
        if (!spirproto::walk_request(b.data(), (long long)b.size(), r, e)) {
            printf("error %d %s\n", e.code, e.what.c_str());
            return 0;
        }
        const long long expected = (long long)r.matrix.rows * r.matrix.columns;
        unsigned flags = 0;
        long long index = 0;
        std::vector<std::string> lines;
        for (const auto &run : r.matrix.runs) {  // the runs end to end; each byte as the decode kernel sees it
            const unsigned char *base = b.data() + run.first;
            const long long bytes = run.second - run.first;
            for (long long off = 0; off < bytes; ++off) {
                if (base[off] & 0x80) {
                    if (off == bytes - 1) flags |= spir::kRunsPast;
                    continue;
                }
                int length;
                const uint64_t v = spir::varint_ending(base, 0, off, length);
                if (length > spir::kVarintMax) flags |= spir::kLongVarint;
                if (word32 && (v >> 32)) flags |= spir::kScalarRange;
                if (index < expected) {
                    const long long at = spir::request_digit_at(index, columns, row_base, col_tiles);
                    uint64_t w = 0;  // the value the digits carry
                    for (int k = 0; k < spir::digits(ct); ++k) w |= (uint64_t)spir::query_digit(v, ct, k) << (8 * k);
                    lines.push_back(std::to_string(at) + " " + std::to_string(w));
                }
                ++index;
            }
        }
        if (index != expected) flags |= spir::kWrongCount;
        printf("flags %u\n", flags);
        for (const std::string &l : lines) printf("%s\n", l.c_str());
        return 0;
    }
    if (cmd == "encode" && argc >= 5) {
        const uint64_t rows = strtoull(argv[2], nullptr, 10), columns = strtoull(argv[3], nullptr, 10);
        const int ct = atoi(argv[4]);
        std::vector<uint64_t> acc;
        for (int i = 5; i < argc; ++i) acc.push_back(strtoull(argv[i], nullptr, 10));
        uint64_t data = 0;  // proto_length_kernel's sum
        for (uint64_t v : acc) data += spir::varint_bytes(spir::finish(v, ct));
        std::vector<unsigned char> out(spir::response_capacity(rows, columns, ct) + 16);
        const int header = spir::response_header(rows, columns, data, out.data());  // proto_write_kernel's thread 0
        if (header != spir::response_header(rows, columns, data, nullptr)) return 3;
        size_t at = (size_t)header;
        for (uint64_t v : acc) at += spir::put_varint(out.data() + at, spir::finish(v, ct));
        for (size_t i = 0; i < at; ++i) printf("%02x", out[i]);
        printf("%s\n%llu\n", at ? "" : ".", (unsigned long long)spir::response_capacity(rows, columns, ct));
        return 0;
    }
    return 2;
}
