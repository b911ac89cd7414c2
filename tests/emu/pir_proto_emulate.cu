// Host replay of the PIR protobuf messages: the walks, offset tables and response template of
// swift-homomorphic-encryption_b200/csrc/pir_proto.hpp (and the walker of protobuf.hpp), evaluated on the CPU, with the
// framing the device writes (response_frame_kernel, pir.cu) replayed from the same template.
//
//   query <n> <bits...>          stdin: an EncryptedIndices as hex; with $EXPECT = "<indices> <ciphertexts>" also
//                                check_query against that shape
//        -> "error <code> <what>", or "ok <num_pir_calls> <count>" then per ciphertext "seeded <poly0> <seed>" or
//           "full <poly0> <poly1> <skip0> <skip1>" (byte offsets into the message)
//   key <n> <count> <bits...>    stdin: a SerializedEvaluationKey as hex (count ciphertexts per key)
//        -> "error ...", or "ok <relin>", then "relin <poly0>:<seed> ..." and one "galois <element> <poly0>:<seed> ..."
//           per map entry in message order
//   request                      stdin: a PIRRequest as hex
//        -> "error ...", or "ok" and every field of hecuda_pir_request_fields
//   response <indices> <chunks> <bytes0> <bytes1> <skip0> <skip1>
//                                stdin: the reply polys back to back (indices x chunks x (bytes0 + bytes1)) as hex
//        -> the PIRResponse, framed from the template and each poly placed at poly_at, as hex
//   read <n> <bits> <indices> <chunks> <skip0> <skip1>   stdin: a PIRResponse as hex
//        -> "error ...", or "ok" and the offset of every reply ciphertext's poly 0
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/pir_proto.hpp"

using namespace hecuda;

static std::vector<unsigned char> read_hex() {
    std::string hex;
    std::cin >> hex;
    if (hex == ".") hex.clear();
    std::vector<unsigned char> out(hex.size() / 2);
    for (size_t i = 0; i < out.size(); ++i) out[i] = (unsigned char)std::stoi(hex.substr(2 * i, 2), nullptr, 16);
    return out;
}

static pirproto::PolySizes sizes(int n, char **bits, int count) {
    pirproto::PolySizes sz;
    sz.n = n;
    for (int i = 0; i < count; ++i) sz.bits.push_back(atoi(bits[i]));
    return sz;
}

static int refuse(const pirproto::Error &e) {
    printf("error %d %s\n", e.code, e.what.c_str());
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const std::string mode = argv[1];
    std::vector<unsigned char> b = read_hex();
    const unsigned char *p = b.empty() ? nullptr : b.data();
    pirproto::Error e;
    if (mode == "query") {
        const pirproto::PolySizes sz = sizes(atoi(argv[2]), argv + 3, argc - 3);
        pirproto::Query q;
        if (!pirproto::walk_encrypted_indices(p, 0, (long long)b.size(), sz, q, e)) return refuse(e);
        const char *check = getenv("EXPECT");  // "<num_pir_calls> <ciphertexts>": check_query against the parameter
        unsigned long long want_indices = 0, want_cts = 0;
        if (check && sscanf(check, "%llu %llu", &want_indices, &want_cts) == 2 &&
            !pirproto::check_query(q, want_indices, (size_t)want_cts, e))
            return refuse(e);
        printf("ok %llu %zu\n", (unsigned long long)q.indices, q.cts.size());
        for (const pirproto::Ciphertext &ct : q.cts)
            if (ct.full)
                printf("full %lld %lld %d %d\n", ct.poly[0], ct.poly[1], ct.skip[0], ct.skip[1]);
            else
                printf("seeded %lld %lld\n", ct.poly[0], ct.seed);
    } else if (mode == "key") {
        const pirproto::PolySizes sz = sizes(atoi(argv[2]), argv + 4, argc - 4);
        pirproto::EvaluationKey k;
        if (!pirproto::walk_evaluation_key(p, 0, (long long)b.size(), sz, atoi(argv[3]), k, e)) return refuse(e);
        printf("ok %d\n", (int)k.relin);
        if (k.relin) {
            printf("relin");
            for (const pirproto::Ciphertext &ct : k.relin_cts) printf(" %lld:%lld", ct.poly[0], ct.seed);
            printf("\n");
        }
        for (const pirproto::GaloisKey &g : k.galois) {
            printf("galois %llu", (unsigned long long)g.element);
            for (const pirproto::Ciphertext &ct : g.cts) printf(" %lld:%lld", ct.poly[0], ct.seed);
            printf("\n");
        }
    } else if (mode == "request") {
        hecuda_pir_request_fields r;
        if (!pirproto::walk_pir_request(p, (long long)b.size(), r, e)) return refuse(e);
        printf("ok\nshard_index %u\nshard_id %d %llu %llu\nconfiguration_hash %llu %llu\nquery %d %llu %llu\n"
               "evaluation_key %d %llu %llu\nkey_metadata %d %llu %llu %llu\n",
               r.shard_index, r.has_shard_id, (unsigned long long)r.shard_id_offset, (unsigned long long)r.shard_id_bytes,
               (unsigned long long)r.configuration_hash_offset, (unsigned long long)r.configuration_hash_bytes, r.has_query,
               (unsigned long long)r.query_offset, (unsigned long long)r.query_bytes, r.has_evaluation_key,
               (unsigned long long)r.evaluation_key_offset, (unsigned long long)r.evaluation_key_bytes, r.has_key_metadata,
               (unsigned long long)r.key_timestamp, (unsigned long long)r.key_identifier_offset,
               (unsigned long long)r.key_identifier_bytes);
    } else if (mode == "response") {
        const long long indices = atoll(argv[2]), chunks = atoll(argv[3]), b0 = atoll(argv[4]), b1 = atoll(argv[5]);
        const pirproto::ResponseLayout rl = pirproto::place_response(indices, chunks, b0, b1, atoi(argv[6]), atoi(argv[7]));
        std::vector<unsigned char> out((size_t)rl.size, 0xee);  // every byte must be written
        for (long long r = 0; r < indices * chunks; ++r) {
            rl.frame(r, [&](long long at, const pirproto::Bytes &bytes) { std::copy(bytes.begin(), bytes.end(), out.begin() + at); });
            for (int q = 0; q < 2; ++q)
                memcpy(out.data() + rl.poly_at(r, q), p + r * (b0 + b1) + (q ? b0 : 0), (size_t)(q ? b1 : b0));
        }
        for (unsigned char c : out) printf("%02x", c);
        printf("\n");
    } else if (mode == "read") {
        const pirproto::PolySizes sz = sizes(atoi(argv[2]), argv + 3, 1);
        std::vector<long long> at;
        if (!pirproto::walk_pir_response(p, (long long)b.size(), sz, atoll(argv[4]), atoll(argv[5]), atoi(argv[6]),
                                         atoi(argv[7]), at, e))
            return refuse(e);
        printf("ok");
        for (long long a : at) printf(" %lld", a);
        printf("\n");
    } else {
        return 2;
    }
    return 0;
}
