// Host replay of the PNNS protobuf messages and query plan: the walks, refusals and response template of
// swift-homomorphic-encryption_b200/csrc/pnns_proto.hpp and the plan of pnns_plan.hpp, evaluated on the CPU, with the
// framing the device writes (launch_frame_runs, proto_respond.cu) replayed from the same runs.
//
//   plan <n> <rows> <columns> <db_rows> <elements...>
//        -> "error <what>", or "ok <ciphertexts> <column_step>", one "row <index> <rotations> <mask as 0/1 digits>" per
//           query row (rows > 1), then "pack <steps...>"
//   request                      stdin: a PNNSRequest as hex
//        -> "error <code> <what>", or "ok" and every field of hecuda_pnns_request_fields, "indices ..." and "ids ..."
//           (each id as offset:length)
//   query <n> <contexts> <columns> <bits...>   stdin: a PNNSRequest as hex
//        -> "error <code> <what>", or "ok <rows>" then per matrix "matrix <count>" and per ciphertext
//           "seeded <poly0> <seed>" or "full <poly0> <poly1> <skip0> <skip1>" (byte offsets into the message)
//   response <replies> <rows> <columns> <ids> <metadata> <contexts> then per context <bytes0> <bytes1> <skip0> <skip1>
//                                <ids>: comma-separated or "-"; <metadata>: comma-separated hex, "~" for an empty
//                                element, or "-" for none.  stdin: every reply poly back to back (context-major) as hex
//        -> the PNNSShardResponse, framed from the runs and each poly placed at poly_at, as hex
//   read <n> <bits> <contexts>   stdin: a PNNSShardResponse as hex
//        -> "error ...", or "ok <rows> <columns> <replies>", per matrix "matrix <skip0> <skip1> <poly0 offsets...>",
//           "ids ..." and "metadata <offset:length>..."
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/pnns_plan.hpp"
#include "../../swift-homomorphic-encryption_b200/csrc/pnns_proto.hpp"

using namespace hecuda;

static std::vector<unsigned char> from_hex(const std::string &hex) {
    std::vector<unsigned char> out(hex.size() / 2);
    for (size_t i = 0; i < out.size(); ++i) out[i] = (unsigned char)std::stoi(hex.substr(2 * i, 2), nullptr, 16);
    return out;
}

static std::vector<unsigned char> read_hex() {
    std::string hex;
    std::cin >> hex;
    if (hex == ".") hex.clear();
    return from_hex(hex);
}

static std::vector<std::string> split(const std::string &s) {
    std::vector<std::string> out;
    if (s == "-") return out;
    std::stringstream ss(s);
    std::string item;
    while (std::getline(ss, item, ',')) out.push_back(item);
    return out;
}

static int refuse(const pnnsproto::Error &e) {
    printf("error %d %s\n", e.code, e.what.c_str());
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const std::string mode = argv[1];
    if (mode == "plan") {
        const long long n = atoll(argv[2]), rows = atoll(argv[3]), columns = atoll(argv[4]), db_rows = atoll(argv[5]);
        std::set<uint64_t> elements;
        for (int i = 6; i < argc; ++i) elements.insert(strtoull(argv[i], nullptr, 10));
        pnnsplan::QueryPlan p;
        std::string err;
        if (!pnnsplan::plan_query(n, rows, columns, db_rows, elements, p, err)) {
            printf("error %s\n", err.c_str());
            return 0;
        }
        printf("ok %lld %d\n", (long long)p.ciphertexts, p.column_step);
        for (long long r = 0; r < rows && rows > 1; ++r) {
            std::string mask;
            for (long long k = 0; k < n; ++k) mask += (char)('0' + p.mask_values[(size_t)(r * n + k)]);
            printf("row %d %d %s\n", p.index[(size_t)r], p.rotate[(size_t)r], mask.c_str());
        }
        printf("pack");
        for (int32_t s : p.pack) printf(" %d", s);
        printf("\n");
        return 0;
    }
    std::vector<unsigned char> b = read_hex();
    const unsigned char *p = b.empty() ? nullptr : b.data();
    pnnsproto::Error e;
    if (mode == "request") {
        pnnsproto::Request r;
        if (!pnnsproto::walk_pnns_request(p, (long long)b.size(), r, e)) return refuse(e);
        const hecuda_pnns_request_fields &f = r.fields;
        printf("ok\n%d %u %d %d %lld %lld %llu %llu %llu %llu %llu %llu %llu\n", f.query_count, f.query_row_count,
               f.has_evaluation_key, f.has_key_metadata, (long long)f.shard_index_count, (long long)f.shard_id_count,
               (unsigned long long)f.config_id_offset, (unsigned long long)f.config_id_bytes,
               (unsigned long long)f.evaluation_key_offset, (unsigned long long)f.evaluation_key_bytes,
               (unsigned long long)f.key_timestamp, (unsigned long long)f.key_identifier_offset,
               (unsigned long long)f.key_identifier_bytes);
        printf("indices");
        for (uint64_t v : r.shard_indices) printf(" %llu", (unsigned long long)v);
        printf("\nids");
        for (const auto &s : r.shard_ids) printf(" %lld:%lld", s.first, s.second - s.first);
        printf("\n");
        return 0;
    }
    if (mode == "query") {
        const long long n = atoll(argv[2]);
        const int contexts = atoi(argv[3]);
        const uint64_t columns = strtoull(argv[4], nullptr, 10);
        pnnsproto::PolySizes sz;
        sz.n = n;
        for (int i = 5; i < argc; ++i) sz.bits.push_back(atoi(argv[i]));
        std::vector<pnnsproto::PolySizes> sizes((size_t)contexts, sz);
        pnnsproto::Request r;
        std::vector<pnnsproto::Matrix> q;
        if (!pnnsproto::walk_pnns_request(p, (long long)b.size(), r, e) || !pnnsproto::walk_query(p, r, sizes, columns, q, e))
            return refuse(e);
        printf("ok %llu\n", (unsigned long long)q[0].rows);
        for (const auto &m : q) {
            printf("matrix %zu\n", m.cts.size());
            for (const auto &ct : m.cts) {
                if (ct.full)
                    printf("full %lld %lld %d %d\n", ct.poly[0], ct.poly[1], ct.skip[0], ct.skip[1]);
                else
                    printf("seeded %lld %lld\n", ct.poly[0], ct.seed);
            }
        }
        return 0;
    }
    if (mode == "response") {
        const long long replies = atoll(argv[2]);
        const uint64_t rows = strtoull(argv[3], nullptr, 10), columns = strtoull(argv[4], nullptr, 10);
        std::vector<uint64_t> ids;
        for (const auto &s : split(argv[5])) ids.push_back(strtoull(s.c_str(), nullptr, 10));
        std::vector<unsigned char> metadata;
        std::vector<uint64_t> offsets{0};
        for (const auto &s : split(argv[6])) {
            const std::vector<unsigned char> m = s == "~" ? std::vector<unsigned char>{} : from_hex(s);
            metadata.insert(metadata.end(), m.begin(), m.end());
            offsets.push_back(metadata.size());
        }
        const int contexts = atoi(argv[7]);
        std::vector<std::array<long long, 2>> bytes;
        std::vector<std::array<int, 2>> skips;
        for (int k = 0; k < contexts; ++k) {
            bytes.push_back({atoll(argv[8 + 4 * k]), atoll(argv[9 + 4 * k])});
            skips.push_back({atoi(argv[10 + 4 * k]), atoi(argv[11 + 4 * k])});
        }
        const pnnsproto::ShardLayout sl =
            pnnsproto::place_shard_response(bytes, skips, replies, rows, columns, ids.data(), (long long)ids.size(),
                                            metadata.data(), offsets.data(), (long long)offsets.size() - 1);
        std::vector<unsigned char> out((size_t)sl.size, 0xEE);
        sl.frame([&](long long at, const pnnsproto::Bytes &run) { std::copy(run.begin(), run.end(), out.begin() + at); });
        size_t from = 0;
        for (int k = 0; k < contexts; ++k)
            for (long long r = 0; r < replies; ++r)
                for (int q = 0; q < 2; ++q) {
                    std::copy(b.begin() + from, b.begin() + from + bytes[(size_t)k][q], out.begin() + sl.poly_at((size_t)k, r, q));
                    from += (size_t)bytes[(size_t)k][q];
                }
        for (unsigned char c : out) printf("%02x", c);
        printf("\n");
        return 0;
    }
    if (mode == "read") {
        pnnsproto::PolySizes sz;
        sz.n = atoll(argv[2]);
        sz.bits.push_back(atoi(argv[3]));
        std::vector<pnnsproto::PolySizes> sizes((size_t)atoi(argv[4]), sz);
        pnnsproto::ShardResponse r;
        if (!pnnsproto::walk_shard_response(p, (long long)b.size(), sizes, r, e)) return refuse(e);
        printf("ok %llu %llu %lld\n", (unsigned long long)r.rows, (unsigned long long)r.columns, r.replies);
        for (size_t k = 0; k < r.poly_at.size(); ++k) {
            printf("matrix %d %d", r.skip[k][0], r.skip[k][1]);
            for (long long at : r.poly_at[k]) printf(" %lld", at);
            printf("\n");
        }
        printf("ids");
        for (uint64_t v : r.ids) printf(" %llu", (unsigned long long)v);
        printf("\nmetadata");
        for (const auto &m : r.metadata) printf(" %lld:%lld", m.first, m.second - m.first);
        printf("\n");
        return 0;
    }
    return 2;
}
