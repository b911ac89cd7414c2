// CPU replay of the OPRF client's device code (csrc/p384.cuh, csrc/aes_gcm.cuh): the same __host__ __device__
// functions blind_kernel, verify_kernel, unblind_kernel and open_kernel call.  Built with nvcc for the host by
// tests/test_oprf_client_emulation.py.
//
// stdin: one operation per line, arguments in hex ("." = empty), integers as big-endian hex; stdout: one line each.
//   ninv a                       -> a^-1 mod n
//   blind r msg                  -> Ser(r HashToGroup(msg))
//   verify pk B response         -> "1" when the proof verifies, "0" when not, "invalid" for an undecodable pk, B or D
//   finalize r D msg             -> the 48-byte Finalize output with N = r^-1 D
//   open key24 nonce12 sealed    -> "1 plaintext" or "0 zeros" (sealed = ciphertext || tag, at least 16 bytes)
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/aes_gcm.cuh"
#include "../../swift-homomorphic-encryption_b200/csrc/p384.cuh"

using namespace hecuda;

static std::vector<unsigned char> unhex(const std::string &s) {
    std::vector<unsigned char> out;
    if (s == ".") return out;
    for (size_t i = 0; i + 1 < s.size(); i += 2) out.push_back((unsigned char)std::stoi(s.substr(i, 2), nullptr, 16));
    return out;
}

static void print_hex(const unsigned char *p, size_t n) {
    if (n == 0) printf(".");
    for (size_t i = 0; i < n; ++i) printf("%02x", p[i]);
}

static p384::Fe plain(const std::string &hex) {  // 48-byte big-endian integer
    std::vector<unsigned char> b = unhex(hex);
    std::vector<unsigned char> padded(48 - b.size(), 0);
    padded.insert(padded.end(), b.begin(), b.end());
    p384::Fe r;
    p384::from_bytes(r, padded.data());
    return r;
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op, a, b, c;
        in >> op >> a >> b >> c;
        if (op == "ninv") {
            p384::Fe r;
            p384::inv_mod_n(r, plain(a));
            unsigned char out[48];
            p384::to_bytes(out, r);
            print_hex(out, 48);
        } else if (op == "blind") {
            const std::vector<unsigned char> msg = unhex(b);
            unsigned char out[p384::kElementBytes];
            p384::blind(out, plain(a), msg.data(), (long long)msg.size());
            print_hex(out, sizeof(out));
        } else if (op == "verify") {
            const std::vector<unsigned char> pk_ser = unhex(a), blinded = unhex(b), response = unhex(c);
            p384::Point pk, pb, pd;
            if (!p384::decompress(pk, pk_ser.data()) || !p384::decompress(pb, blinded.data()) ||
                !p384::decompress(pd, response.data())) {
                printf("invalid");
            } else {
                unsigned char seed[p384::kSeedBytes];
                p384::composite_seed(seed, pk_ser.data());
                printf("%d", (int)p384::verify_proof(pk, pk_ser.data(), seed, pb, blinded.data(), pd, response.data(),
                                                     response.data() + p384::kElementBytes));
            }
        } else if (op == "finalize") {
            const std::vector<unsigned char> evaluated = unhex(b), msg = unhex(c);
            p384::Point d;
            if (!p384::decompress(d, evaluated.data())) return 3;
            unsigned char out[p384::kOutputBytes];
            p384::unblind_finalize(out, plain(a), d, msg.data(), (long long)msg.size());
            print_hex(out, sizeof(out));
        } else if (op == "open") {
            const std::vector<unsigned char> key = unhex(a), nonce = unhex(b), sealed = unhex(c);
            unsigned char sbox[256];
            drbg::u32w te0[256], words[6], rk[gcm::kRoundKeyWords192];
            drbg::make_tables(sbox, te0);
            for (int w = 0; w < 6; ++w)
                words[w] = ((drbg::u32w)key[4 * w] << 24) | ((drbg::u32w)key[4 * w + 1] << 16) |
                           ((drbg::u32w)key[4 * w + 2] << 8) | key[4 * w + 3];
            gcm::expand_key_192(words, rk, sbox);
            const long long len = (long long)sealed.size() - 16;
            std::vector<unsigned char> out(len + 1, 0xee);
            const bool ok = gcm::open(rk, te0, sbox, nonce.data(), sealed.data(), len, sealed.data() + len, out.data());
            printf("%d ", (int)ok);
            print_hex(out.data(), (size_t)len);
        } else {
            return 2;
        }
        printf("\n");
    }
    return 0;
}
