// CPU replay of the OPRF server's device code (csrc/p384.cuh): the same __host__ __device__ functions
// proof_setup_kernel, blind_evaluate_kernel and proof_kernel call.  Built with nvcc for the host by
// tests/test_oprf_server_emulation.py.
//
// stdin: one operation per line, arguments in hex, integers as big-endian hex; stdout: one line each.
//   nmul a b | nadd a b | nsub a b   -> a b, a + b, a - b mod n (a < 2^384 for nmul, else a, b < n)
//   nreduce72 bytes                  -> the 72-byte integer mod n
//   h2s msg                          -> HashToScalar(msg)
//   recode k                         -> the 97 recoding bytes as signed decimals
//   smulct k x y                     -> compressed k (x, y) through scalar_mul_ct
//   decompress bytes                 -> "x y" (affine) or "invalid"
//   composite seed48 B D             -> d0
//   nonce k seed32 B                 -> r
//   prove k r B                      -> the 145-byte response with nonce r, or "invalid"
//   respond k seed32 B               -> the 145-byte response with the derived nonce, or "invalid"
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/p384.cuh"

using namespace hecuda;

static std::vector<unsigned char> unhex(const std::string &s) {
    std::vector<unsigned char> out;
    if (s == ".") return out;
    for (size_t i = 0; i + 1 < s.size(); i += 2) out.push_back((unsigned char)std::stoi(s.substr(i, 2), nullptr, 16));
    return out;
}

static void print_hex(const unsigned char *p, size_t n) {
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

static void print_plain(const p384::Fe &a) {
    unsigned char b[48];
    p384::to_bytes(b, a);
    print_hex(b, 48);
}

static void print_fe(const p384::Fe &m) {  // Montgomery form in, plain out
    p384::Fe a;
    p384::from_mont(a, m);
    print_plain(a);
}

// the response with nonce r (derived from seed32 when r is null); false for an invalid query or r = 0
static bool respond(unsigned char out[p384::kResponseBytes], const p384::Fe &k, const p384::Fe *r_given,
                    const std::vector<unsigned char> &seed32, const std::vector<unsigned char> &query) {
    signed char digits[p384::kDigits + 1];
    p384::recode_scalar(k, digits);
    p384::Point g, pk;
    p384::generator(g);
    p384::scalar_mul(pk, g, digits);
    unsigned char setup[p384::kElementBytes + p384::kSeedBytes];
    p384::compress(setup, pk);
    p384::composite_seed(setup + p384::kElementBytes, setup);
    p384::Fe mx, my, r;
    if (!p384::blind_evaluate_composite(out, mx, my, query.data(), digits, setup + p384::kElementBytes)) return false;
    if (r_given) {
        r = *r_given;
    } else {
        p384::proof_nonce(r, k, seed32.data(), query.data());
    }
    if (p384::is_zero(r)) return false;
    p384::generate_proof(out + p384::kElementBytes, digits, k, setup, mx, my, r);
    return true;
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op, a, b, c;
        in >> op >> a >> b >> c;
        if (op == "nmul") {
            p384::Fe r;
            p384::mul_mod_n(r, plain(a), plain(b));
            print_plain(r);
        } else if (op == "nadd" || op == "nsub") {
            p384::Fe r;
            if (op == "nadd") p384::add<p384::ModN>(r, plain(a), plain(b));
            if (op == "nsub") p384::sub<p384::ModN>(r, plain(a), plain(b));
            print_plain(r);
        } else if (op == "nreduce72") {
            const std::vector<unsigned char> m = unhex(a);
            p384::Fe r;
            p384::from_bytes72_mod_n(r, m.data());
            print_plain(r);
        } else if (op == "h2s") {
            const std::vector<unsigned char> m = unhex(a);
            sha512::Sha384 s;
            p384::xmd_begin(s);
            s.bytes(m.data(), (long long)m.size());
            p384::Fe r;
            p384::hash_to_scalar_finish(r, s);
            print_plain(r);
        } else if (op == "recode") {
            signed char digits[p384::kDigits + 1];
            p384::recode_scalar(plain(a), digits);
            for (int i = 0; i <= p384::kDigits; ++i) printf(i ? " %d" : "%d", digits[i]);
        } else if (op == "smulct") {
            signed char digits[p384::kDigits + 1];
            p384::recode_scalar(plain(a), digits);
            p384::Point p, r;
            p384::to_mont(p.x, plain(b));
            p384::to_mont(p.y, plain(c));
            p.z = p384::kOneHost;
            p384::scalar_mul_ct(r, p, digits);
            unsigned char out[p384::kElementBytes];
            p384::compress(out, r);
            print_hex(out, sizeof(out));
        } else if (op == "decompress") {
            const std::vector<unsigned char> m = unhex(a);
            p384::Point p;
            if (m.size() == p384::kElementBytes && p384::decompress(p, m.data())) {
                print_fe(p.x);
                printf(" ");
                print_fe(p.y);
            } else {
                printf("invalid");
            }
        } else if (op == "composite") {
            const std::vector<unsigned char> seed = unhex(a), blinded = unhex(b), evaluated = unhex(c);
            p384::Fe d0;
            p384::composite_scalar(d0, seed.data(), blinded.data(), evaluated.data());
            print_plain(d0);
        } else if (op == "nonce") {
            const std::vector<unsigned char> seed = unhex(b), query = unhex(c);
            p384::Fe r;
            p384::proof_nonce(r, plain(a), seed.data(), query.data());
            print_plain(r);
        } else if (op == "prove" || op == "respond") {
            const p384::Fe k = plain(a), r = plain(b);
            const std::vector<unsigned char> seed = unhex(b), query = unhex(c);
            unsigned char out[p384::kResponseBytes];
            if (respond(out, k, op == "prove" ? &r : nullptr, seed, query)) {
                print_hex(out, sizeof(out));
            } else {
                printf("invalid");
            }
        } else {
            return 2;
        }
        printf("\n");
    }
    return 0;
}
