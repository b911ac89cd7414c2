// Host replay of saving and loading processed PNNS databases: the protobuf walker and writer of
// swift-homomorphic-encryption_b200/csrc/pnns_database_io.hpp, the chunk planner of database_io.hpp, and the
// per-plaintext offset map (tagged_rows_offset with the framing length) that the codec kernels use, evaluated on the CPU.
//
//   walk                stdin: a SerializedProcessedDatabase as hex
//        -> "error <code> <what>", or "ok", then one "matrix <rows> <cols> <packing> <dim> <baby> <giant> <count>"
//           and one "polys <offset>:<bytes> ..." line per matrix, "ids ...", "metadata <offset>:<bytes> ...", "config ..."
//   resave <budget>     stdin: the same; walks it, places a serialization of what it found with the library's writer,
//                       frames every plaintext as the serialize kernels do (chunk by chunk, at most `budget` bytes)
//                       and copies each poly from the input
//        -> "chunks <count>", then the new file as hex
//   server | client     stdin: a ServerConfig / ClientConfig message as hex
//        -> "error <code> <what>", or "config ..." and the message written back as hex
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/database_io.hpp"
#include "../../swift-homomorphic-encryption_b200/csrc/kernels.cuh"
#include "../../swift-homomorphic-encryption_b200/csrc/pnns_database_io.hpp"

using namespace hecuda;

static std::vector<unsigned char> read_hex() {
    std::string hex;
    std::cin >> hex;
    if (hex == ".") hex.clear();
    std::vector<unsigned char> out;
    for (size_t k = 0; k + 1 < hex.size(); k += 2) out.push_back((unsigned char)strtoul(hex.substr(k, 2).c_str(), nullptr, 16));
    return out;
}

static std::string to_hex(const std::vector<unsigned char> &bytes) {
    static const char *digits = "0123456789abcdef";
    std::string out;
    for (unsigned char b : bytes) out += std::string(1, digits[b >> 4]) + digits[b & 15];
    return out;
}

static void print_config(const hecuda_pnns_server_config &c) {
    printf("config %llu %llu %d", (unsigned long long)c.poly_degree, (unsigned long long)c.plaintext_modulus,
           c.coefficient_moduli_count);
    for (int k = 0; k < c.coefficient_moduli_count; ++k) printf(" %llu", (unsigned long long)c.coefficient_moduli[k]);
    printf(" %d %d %d %llu %d %u %u %u %u %d", c.error_std_dev, c.security_level, c.he_scheme,
           (unsigned long long)c.scaling_factor, c.query_packing, c.query_vector_dimension, c.query_baby_step,
           c.query_giant_step, c.vector_dimension, c.galois_element_count);
    for (int k = 0; k < c.galois_element_count; ++k) printf(" %u", c.galois_elements[k]);
    printf(" %d %d", c.distance_metric, c.extra_plaintext_moduli_count);
    for (int k = 0; k < c.extra_plaintext_moduli_count; ++k) printf(" %llu", (unsigned long long)c.extra_plaintext_moduli[k]);
    printf(" %d %u %u %u\n", c.database_packing, c.database_vector_dimension, c.database_baby_step, c.database_giant_step);
}

static bool walk(const std::vector<unsigned char> &file, pnnsio::Database &db) {
    pnnsio::Error e;
    if (!pnnsio::walk_database(file.data(), (long long)file.size(), db, e)) {
        printf("error %d %s\n", e.code, e.what.c_str());
        return false;
    }
    return true;
}

static int run_walk() {
    const std::vector<unsigned char> file = read_hex();
    pnnsio::Database db;
    if (!walk(file, db)) return 0;
    puts("ok");
    for (const pnnsio::Matrix &m : db.matrices) {
        printf("matrix %lld %lld %d %u %u %u %zu\npolys", m.rows, m.cols, m.packing, m.bsgs[0], m.bsgs[1], m.bsgs[2],
               m.poly_at.size());
        for (size_t p = 0; p < m.poly_at.size(); ++p) printf(" %lld:%lld", m.poly_at[p], m.poly_bytes[p]);
        printf("\n");
    }
    printf("ids");
    for (uint64_t v : db.entry_ids) printf(" %llu", (unsigned long long)v);
    printf("\nmetadata");
    for (size_t k = 0; k < db.metadata_at.size(); ++k) printf(" %lld:%lld", db.metadata_at[k], db.metadata_bytes[k]);
    printf("\n");
    print_config(db.config);
    return 0;
}

static int run_resave(long long budget) {
    const std::vector<unsigned char> file = read_hex();
    pnnsio::Database db;
    if (!walk(file, db)) return 0;
    std::vector<pnnsio::MatrixShape> shapes;
    for (const pnnsio::Matrix &m : db.matrices) shapes.push_back({m.rows, m.cols, (long long)m.poly_at.size(), m.poly_bytes.at(0)});
    std::vector<unsigned char> metadata;
    std::vector<uint64_t> offsets{0};
    for (size_t k = 0; k < db.metadata_at.size(); ++k) {
        metadata.insert(metadata.end(), file.begin() + db.metadata_at[k], file.begin() + db.metadata_at[k] + db.metadata_bytes[k]);
        offsets.push_back(metadata.size());
    }
    const pnnsio::Placement pl = pnnsio::place_database(shapes, db.entry_ids.data(), (long long)db.entry_ids.size(),
                                                        metadata.data(), offsets.data(), (long long)db.metadata_at.size(), db.config);
    std::vector<unsigned char> out((size_t)pl.size, 0xee);  // every byte must be written
    long long chunks = 0;
    for (size_t k = 0; k < pl.matrices.size(); ++k) {
        const pnnsio::MatrixPlacement &mp = pl.matrices[k];
        memcpy(out.data() + mp.head_at, mp.head.data(), mp.head.size());
        memcpy(out.data() + mp.tag.back(), mp.tail.data(), mp.tail.size());
        const long long count = (long long)mp.tag.size() - 1;
        for (const dbio::Chunk &ch : dbio::plan_chunks(mp.tag, 0, count, budget)) {
            ++chunks;
            const long long base = mp.tag[(size_t)ch.first];
            std::vector<unsigned char> staged((size_t)(mp.tag[(size_t)(ch.first + ch.count)] - base), 0xee);
            for (long long p = 0; p < ch.count; ++p) {
                // write_tag, then the rows at tagged_rows_offset (here: the input's poly, which the kernels would pack)
                const long long offset = tagged_rows_offset(mp.tag.data() + ch.first, base, p, (int)mp.frame.size());
                memcpy(staged.data() + (mp.tag[(size_t)(ch.first + p)] - base), mp.frame.data(), mp.frame.size());
                const long long src = db.matrices[k].poly_at[(size_t)(ch.first + p)];
                memcpy(staged.data() + offset, file.data() + src, (size_t)db.matrices[k].poly_bytes[(size_t)(ch.first + p)]);
            }
            memcpy(out.data() + base, staged.data(), staged.size());
        }
    }
    memcpy(out.data() + pl.rest_at, pl.rest.data(), pl.rest.size());
    printf("chunks %lld\n%s\n", chunks, to_hex(out).c_str());
    return 0;
}

static int run_config(bool server) {
    const std::vector<unsigned char> bytes = read_hex();
    hecuda_pnns_server_config c{};
    pnnsio::Error e;
    const bool ok = server ? pnnsio::parse_server_config(bytes.data(), 0, (long long)bytes.size(), c, e)
                           : pnnsio::parse_client_config(bytes.data(), 0, (long long)bytes.size(), c, e);
    if (!ok) {
        printf("error %d %s\n", e.code, e.what.c_str());
        return 0;
    }
    print_config(c);
    puts(to_hex(server ? pnnsio::encode_server_config(c) : pnnsio::encode_client_config(c)).c_str());
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    if (!strcmp(argv[1], "walk")) return run_walk();
    if (!strcmp(argv[1], "resave") && argc > 2) return run_resave(atoll(argv[2]));
    if (!strcmp(argv[1], "server")) return run_config(true);
    if (!strcmp(argv[1], "client")) return run_config(false);
    return 2;
}
