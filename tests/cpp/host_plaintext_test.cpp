// host_plaintext_test.cpp -- the plaintext side of the C++ mirror (host/HeScheme.hpp) on a GPU: SIMD encode / decode round
// trips in Coeff and Eval format, ciphertext +- plaintext, and the reference's error paths.  Writes the translated
// ciphertexts for the Python test to compare with the reference restatement.
//   usage: host_plaintext_test <out.bin>     (N = 4096, q = 27/28/28 bits, t = 65537)
#include <cstdio>
#include <fstream>

#include "../../swift-homomorphic-encryption_b200/host/HeScheme.hpp"

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const int64_t n = 4096;
    const std::vector<uint64_t> moduli = {134176769, 268369921, 268361729};
    const uint64_t t = 65537;
    auto ctx = std::make_shared<const he::Context>(n, moduli, t);
    const int L = ctx->ciphertextModuliCount();
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) {
            std::fprintf(stderr, "FAIL: %s\n", what);
            ++failures;
        }
    };
    expect(he::Bfv::supportsSimdEncoding(*ctx), "supportsSimdEncoding");
    std::vector<uint64_t> values(n / 2), padded(n, 0), other(n);
    for (int64_t i = 0; i < n / 2; ++i) padded[i] = values[i] = (uint64_t)(i * 7919 + 13) % t;
    for (int64_t i = 0; i < n; ++i) other[i] = (uint64_t)(i * 104729 + 5) % t;
    const std::vector<uint64_t> pt = he::Bfv::encodeSimd(*ctx, values);
    expect(he::Bfv::decodeSimd(*ctx, pt) == padded, "decode(encode(values))");
    const he::PolyRq ev = he::Bfv::encodeSimd(ctx, values, L);
    expect(he::Bfv::decodeSimd(ev) == padded, "decodeEval(encode(values, moduliCount: L))");

    he::Ciphertext ct(ctx, 2, L);
    for (size_t i = 0; i < ct.data.size(); ++i) ct.data[i] = (uint64_t)(i * 2654435761u) % moduli[(i / n) % L];
    he::Ciphertext added = ct, subtracted = ct;
    const std::vector<uint64_t> pt2 = he::Bfv::encodeSimd(*ctx, other);
    he::Bfv::addAssignCoeff(added, pt2);
    he::Bfv::subAssignCoeff(subtracted, pt2);
    const he::Ciphertext from = he::Bfv::subCoeff(pt2, ct);
    he::Ciphertext back = added;
    he::Bfv::subAssignCoeff(back, pt2);
    expect(back.data == ct.data, "(ct + pt) - pt == ct");

    // errors: correction factor, value >= t, too many values, no SIMD support
    auto throws = [&](auto fn, he::HeError::Kind kind, const char *what) {
        try {
            fn();
            expect(false, what);
        } catch (const he::HeError &e) {
            expect(e.kind == kind, what);
        }
    };
    he::Ciphertext scaled = ct;
    scaled.correctionFactor = 3;
    throws([&] { he::Bfv::addAssignCoeff(scaled, pt2); }, he::HeError::invalidCiphertext, "invalidCorrectionFactor");
    throws([&] { he::Bfv::encodeSimd(*ctx, std::vector<uint64_t>{t}); }, he::HeError::invalidCiphertext, "encodingDataOutOfBounds");
    throws([&] { he::Bfv::encodeSimd(*ctx, std::vector<uint64_t>(n + 1, 0)); }, he::HeError::invalidCiphertext,
           "encodingDataCountExceedsLimit");
    {
        he::Context plain17(n, moduli, 17);
        expect(!he::Bfv::supportsSimdEncoding(plain17), "t = 17 has no SIMD encoding");
        throws([&] { he::Bfv::encodeSimd(plain17, values); }, he::HeError::unsupportedHeOperation, "simdEncodingNotSupported");
    }

    std::ofstream f(argv[1], std::ios::binary);
    const std::vector<const std::vector<uint64_t> *> outputs = {&ct.data, &pt2, &added.data, &subtracted.data, &from.data};
    for (const std::vector<uint64_t> *v : outputs) f.write((const char *)v->data(), (std::streamsize)(8 * v->size()));
    if (failures) return 1;
    std::printf("host plaintext mirror ok\n");
    return 0;
}
