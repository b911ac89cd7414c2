// CPU replay of the symmetric-PIR device code (csrc/p384.cuh, csrc/sha512.cuh, csrc/aes_gcm.cuh): the same
// __host__ __device__ functions oprf_evaluate_kernel and seal_kernel call.  Built with nvcc for the host by
// tests/test_symmetric_pir_emulation.py.
//
// stdin: one operation per line, arguments in hex ("." = empty), integers as big-endian hex; stdout: one line each.
//   sha384 msg              -> digest
//   mul a b | add a b | sub a b | inv a   (a, b < p)  -> result mod p
//   sqrt_ratio u v          -> "1 y" or "0 y"
//   reduce72 bytes          -> the 72-byte integer mod p
//   map u                   -> "x y square" (affine)
//   h2g msg                 -> "x y" of HashToGroup(msg)
//   recode k                -> the 97 recoding bytes (digits, then the flip flag) as signed decimals
//   smul k x y              -> compressed k (x, y)
//   eval k msg              -> the 48-byte OPRF output
//   seal key nonce value    -> AES-GCM-192 ciphertext || tag
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

static p384::Fe mont(const std::string &hex) {
    p384::Fe r;
    p384::to_mont(r, plain(hex));
    return r;
}

static void print_fe(const p384::Fe &m) {  // Montgomery form in, plain big-endian hex out
    p384::Fe a;
    unsigned char b[48];
    p384::from_mont(a, m);
    p384::to_bytes(b, a);
    print_hex(b, 48);
}

static void print_point(const p384::Point &p) {
    p384::Fe x, y;
    if (!p384::to_affine(x, y, p)) {
        printf("inf inf");
        return;
    }
    print_fe(x);
    printf(" ");
    print_fe(y);
}

int main() {
    unsigned char sbox[256];
    drbg::u32w te0[256];
    drbg::make_tables(sbox, te0);
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op, a, b, c;
        in >> op >> a >> b >> c;
        if (op == "sha384") {
            const std::vector<unsigned char> m = unhex(a);
            unsigned char d[48];
            sha512::sha384(m.data(), (long long)m.size(), d);
            print_hex(d, 48);
        } else if (op == "mul" || op == "add" || op == "sub") {
            p384::Fe x = mont(a), y = mont(b), r;
            if (op == "mul") p384::mul(r, x, y);
            if (op == "add") p384::add(r, x, y);
            if (op == "sub") p384::sub(r, x, y);
            print_fe(r);
        } else if (op == "inv") {
            p384::Fe r;
            p384::inv(r, mont(a));
            print_fe(r);
        } else if (op == "sqrt_ratio") {
            p384::Fe y;
            const bool qr = p384::sqrt_ratio(y, mont(a), mont(b));
            printf("%d ", qr ? 1 : 0);
            print_fe(y);
        } else if (op == "reduce72") {
            const std::vector<unsigned char> m = unhex(a);
            p384::Fe r;
            p384::from_bytes72(r, m.data());
            print_fe(r);
        } else if (op == "map") {
            p384::Point p;
            const bool square = p384::map_to_curve(p, mont(a));
            print_point(p);
            printf(" %d", square ? 1 : 0);
        } else if (op == "h2g") {
            const std::vector<unsigned char> m = unhex(a);
            p384::Point p;
            p384::hash_to_group(p, m.data(), (long long)m.size());
            print_point(p);
        } else if (op == "recode") {
            signed char digits[p384::kDigits + 1];
            p384::recode_scalar(plain(a), digits);
            for (int i = 0; i <= p384::kDigits; ++i) printf(i ? " %d" : "%d", digits[i]);
        } else if (op == "smul") {
            signed char digits[p384::kDigits + 1];
            p384::recode_scalar(plain(a), digits);
            p384::Point p{mont(b), mont(c), p384::kOneHost}, r;
            p384::scalar_mul(r, p, digits);
            unsigned char out[p384::kElementBytes];
            p384::compress(out, r);
            print_hex(out, sizeof(out));
        } else if (op == "eval") {
            signed char digits[p384::kDigits + 1];
            p384::recode_scalar(plain(a), digits);
            const std::vector<unsigned char> m = unhex(b);
            unsigned char out[p384::kOutputBytes];
            p384::oprf_evaluate(out, digits, m.data(), (long long)m.size());
            print_hex(out, sizeof(out));
        } else if (op == "seal") {
            const std::vector<unsigned char> key = unhex(a), nonce = unhex(b), value = unhex(c);
            drbg::u32w kw[6], rk[gcm::kRoundKeyWords192];
            for (int i = 0; i < 6; ++i)
                kw[i] = ((drbg::u32w)key[4 * i] << 24) | ((drbg::u32w)key[4 * i + 1] << 16) | ((drbg::u32w)key[4 * i + 2] << 8) |
                        key[4 * i + 3];
            gcm::expand_key_192(kw, rk, sbox);
            std::vector<unsigned char> out(value.size() + 16);
            gcm::seal(rk, te0, sbox, nonce.data(), value.data(), (long long)value.size(), out.data());
            print_hex(out.data(), out.size());
        } else {
            return 2;
        }
        printf("\n");
    }
    return 0;
}
