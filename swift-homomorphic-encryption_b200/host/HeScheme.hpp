// HeScheme.hpp -- C++ host-side mirror of the reference's scheme surface for the RNS-BFV hot path, over the C ABI in
// include/hecuda.h.  The reference's host language (Swift) is not available in this build image; this header keeps
// the reference's names, argument meaning and error behaviour so that callers and tests read like the reference's:
//
//   he::Context                 Context<Bfv<UInt64>>            Sources/HomomorphicEncryption/Context.swift:19,94-143
//   he::PolyRq                  PolyRq<UInt64, F>               PolyRq/PolyRq.swift:21-52   (Array2d data, rows x N)
//   he::Ciphertext              Ciphertext<Bfv<UInt64>, Coeff>  Ciphertext.swift:18-28
//   he::EvaluationKey           EvaluationKey<Bfv<UInt64>>      Keys.swift:222
//   he::Bfv::mulAssign          Bfv.mulAssign                   Bfv/Bfv+Multiply.swift:18-21
//   he::Bfv::relinearize        Bfv.relinearize                 Bfv/Bfv.swift:201-219
//   he::Bfv::modSwitchDown      Bfv.modSwitchDown               Bfv/Bfv.swift:163-171
//   he::Bfv::forwardNtt/inverseNtt  PolyRq.forwardNtt/inverseNtt  PolyRq/PolyRq+Ntt.swift:230,541
//   he::Bfv::encodeSimd/decodeSimd  Bfv.encode / decodeCoeff / decodeEval (.simd)  Encoding.swift:197-245, Bfv+Encode.swift
//   he::Bfv::addAssignCoeff/subAssignCoeff/subCoeff  Bfv.swift:110-117, HeScheme.swift:1540-1542
//   he::HeError                 HeError                         Error.swift:17-54
//
// Batched overloads take a span of ciphertexts so one call saturates the GPU (SURVEY.md section 8b, "Threading").
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/hecuda.h"

namespace he {

class HeError : public std::runtime_error {
   public:
    enum Kind { invalidCiphertext, incompatibleCiphertexts, invalidPolyContext, invalidContext, unsupportedHeOperation,
                missingRelinearizationKey, missingGaloisKey, invalidEncryptionParameters, deviceError };
    HeError(Kind k, const std::string &m) : std::runtime_error(m), kind(k) {}
    Kind kind;
    static HeError fromStatus(int32_t rc) {
        const std::string msg = hecuda_last_error() ? hecuda_last_error() : "";
        switch (rc) {
            case HECUDA_ERR_UNSUPPORTED: return HeError(unsupportedHeOperation, msg);
            case HECUDA_ERR_MISSING_KEY:
                return HeError(msg.find("Galois") != std::string::npos ? missingGaloisKey : missingRelinearizationKey, msg);
            case HECUDA_ERR_INVALID_ARGUMENT: return HeError(invalidCiphertext, msg);
            default: return HeError(deviceError, msg);
        }
    }
};
inline void check(int32_t rc) {
    if (rc != HECUDA_OK) throw HeError::fromStatus(rc);
}

// Context<Bfv<UInt64>>: coefficientModuli = q_0..q_{L-1}, q_ks (Context.swift:102-107)
class Context {
   public:
    Context(int64_t polyDegree, std::vector<uint64_t> coefficientModuli, uint64_t plaintextModulus)
        : degree(polyDegree), coefficientModuli(std::move(coefficientModuli)), plaintextModulus(plaintextModulus) {
        int32_t rc = hecuda_context_create(degree, this->coefficientModuli.data(), (int32_t)this->coefficientModuli.size(),
                                           plaintextModulus, &handle_);
        if (rc != HECUDA_OK) {
            HeError e = HeError::fromStatus(rc);
            throw HeError(rc == HECUDA_ERR_UNSUPPORTED ? HeError::unsupportedHeOperation : HeError::invalidEncryptionParameters,
                          e.what());
        }
    }
    ~Context() { hecuda_context_destroy(handle_); }
    Context(const Context &) = delete;
    Context &operator=(const Context &) = delete;
    int ciphertextModuliCount() const { return (int)coefficientModuli.size() - 1; }
    hecuda_context *handle() const { return handle_; }
    bool operator==(const Context &o) const {  // Context.== (Context.swift:150-152)
        return this == &o || (degree == o.degree && coefficientModuli == o.coefficientModuli && plaintextModulus == o.plaintextModulus);
    }
    const int64_t degree;
    const std::vector<uint64_t> coefficientModuli;
    const uint64_t plaintextModulus;

   private:
    hecuda_context *handle_ = nullptr;
};

// PolyRq: rows x N residues, row-major (Array2d.swift:115-123).  `moduliCount` rows of the ciphertext context.
struct PolyRq {
    std::shared_ptr<const Context> context;
    int moduliCount = 0;
    std::vector<uint64_t> data;
    PolyRq() = default;
    PolyRq(std::shared_ptr<const Context> c, int rows) : context(std::move(c)), moduliCount(rows), data((size_t)rows * context->degree) {}
};

// Ciphertext: polys back to back (Ciphertext.swift:18-28); Bfv's canonical format is Coeff.
struct Ciphertext {
    std::shared_ptr<const Context> context;
    int polyCount = 0, moduliCount = 0;
    uint64_t correctionFactor = 1;
    std::vector<uint64_t> data;  // polyCount x moduliCount x N
    Ciphertext() = default;
    Ciphertext(std::shared_ptr<const Context> c, int polys, int rows)
        : context(std::move(c)), polyCount(polys), moduliCount(rows), data((size_t)polys * rows * context->degree) {}
    size_t polyWords() const { return (size_t)moduliCount * context->degree; }
};

class EvaluationKey {
   public:
    // relinearizationKey: the _KeySwitchKey's L ciphertexts x 2 polys x (L+1) x N in Eval format (Keys.swift:66-99)
    EvaluationKey(std::shared_ptr<const Context> c, const std::vector<uint64_t> &relinearizationKey) : context(std::move(c)) {
        const size_t L = context->ciphertextModuliCount();
        if (relinearizationKey.size() != L * 2 * (L + 1) * (size_t)context->degree)
            throw HeError(HeError::invalidContext, "relinearization key must be L x 2 x (L+1) x N");
        check(hecuda_evk_create(context->handle(), relinearizationKey.data(), &handle_));
    }
    // an evaluation key without a relinearization key (EvaluationKeyConfig.hasRelinearizationKey == false)
    explicit EvaluationKey(std::shared_ptr<const Context> c) : context(std::move(c)) {
        check(hecuda_evk_create_empty(context->handle(), &handle_));
    }
    // GaloisKey.keys[element] (Keys.swift:150-163): L ciphertexts x 2 polys x (L+1) x N, Eval format
    void setGaloisKey(uint32_t element, const std::vector<uint64_t> &key) {
        const size_t L = context->ciphertextModuliCount();
        if (key.size() != L * 2 * (L + 1) * (size_t)context->degree)
            throw HeError(HeError::invalidContext, "Galois key must be L x 2 x (L+1) x N");
        check(hecuda_evk_set_galois_key(handle_, element, key.data()));
    }
    // EvaluationKey(deserialize:context:) (SerializedKeys.swift:141-157) with every key ciphertext
    // .seeded(poly0:seed:): relinPoly0 L x B bytes and relinSeeds L x 32 (both empty: no relinearization key), B =
    // hecuda_poly_serialized_byte_count(BASE_KEYSWITCH, L+1 rows, skipLSBs 0); galoisPoly0 / galoisSeeds hold the same
    // for each of `elements`, in that order.  The seeds are expanded and poly0 unpacked on the device.
    static std::unique_ptr<EvaluationKey> deserialize(std::shared_ptr<const Context> c, const std::vector<uint8_t> &relinPoly0,
                                                      const std::vector<uint8_t> &relinSeeds,
                                                      const std::vector<uint32_t> &elements,
                                                      const std::vector<uint8_t> &galoisPoly0,
                                                      const std::vector<uint8_t> &galoisSeeds) {
        const size_t L = c->ciphertextModuliCount();
        uint64_t bytes = 0;
        check(hecuda_poly_serialized_byte_count(c->handle(), HECUDA_BASE_KEYSWITCH, (int32_t)L + 1, 0, &bytes));
        const bool relin = !relinPoly0.empty() || !relinSeeds.empty();
        if (relin && (relinPoly0.size() != L * bytes || relinSeeds.size() != L * 32))
            throw HeError(HeError::invalidContext, "serializedBufferSizeMismatch: relinearization key must be L x B and L x 32 bytes");
        if (galoisPoly0.size() != elements.size() * L * bytes || galoisSeeds.size() != elements.size() * L * 32)
            throw HeError(HeError::invalidContext, "serializedBufferSizeMismatch: Galois keys must be L x B and L x 32 bytes each");
        hecuda_evk *h = nullptr;
        check(hecuda_evk_create_serialized(c->handle(), relin ? relinPoly0.data() : nullptr, relin ? relinSeeds.data() : nullptr,
                                           elements.data(), (int32_t)elements.size(), galoisPoly0.data(), galoisSeeds.data(), &h));
        return std::unique_ptr<EvaluationKey>(new EvaluationKey(std::move(c), h));
    }
    ~EvaluationKey() { hecuda_evk_destroy(handle_); }
    EvaluationKey(const EvaluationKey &) = delete;
    EvaluationKey &operator=(const EvaluationKey &) = delete;
    std::shared_ptr<const Context> context;
    hecuda_evk *handle() const { return handle_; }

   private:
    EvaluationKey(std::shared_ptr<const Context> c, hecuda_evk *h) : context(std::move(c)), handle_(h) {}
    hecuda_evk *handle_ = nullptr;
};

// enum Bfv<UInt64>: HeScheme -- the hot-path statics
struct Bfv {
    static constexpr int freshCiphertextPolyCount = 2;  // HeScheme.freshCiphertextPolyCount

    // validateEquality + the guards of multiplyWithoutScaling (Bfv+Multiply.swift:66-76)
    static void validateMultiply(const Ciphertext &lhs, const Ciphertext &rhs) {
        if (!lhs.context || !rhs.context || !(*lhs.context == *rhs.context))
            throw HeError(HeError::invalidContext, "ciphertexts have different contexts");
        if (lhs.polyCount != freshCiphertextPolyCount || lhs.correctionFactor != 1)
            throw HeError(HeError::invalidCiphertext, "lhs must have 2 polys and correction factor 1");
        if (rhs.polyCount != freshCiphertextPolyCount || rhs.correctionFactor != 1)
            throw HeError(HeError::invalidCiphertext, "rhs must have 2 polys and correction factor 1");
        if (lhs.moduliCount != rhs.moduliCount) throw HeError(HeError::incompatibleCiphertexts, "different poly contexts");
        if (lhs.moduliCount != lhs.context->ciphertextModuliCount())
            throw HeError(HeError::unsupportedHeOperation, "ct x ct multiply is supported at the top level only");
    }

    // lhs *= rhs  ->  lhs becomes a 3-poly ciphertext
    static void mulAssign(Ciphertext &lhs, const Ciphertext &rhs) {
        validateMultiply(lhs, rhs);
        Ciphertext out(lhs.context, 3, lhs.moduliCount);
        check(hecuda_bfv_multiply(lhs.context->handle(), lhs.data.data(), rhs.data.data(), out.data.data(), 1));
        lhs = std::move(out);
    }
    // batched: lhs[i] *= rhs[i] for all i in one device pass
    static void mulAssign(std::vector<Ciphertext> &lhs, const std::vector<Ciphertext> &rhs) {
        if (lhs.size() != rhs.size()) throw HeError(HeError::incompatibleCiphertexts, "batch sizes differ");
        if (lhs.empty()) return;
        for (size_t i = 0; i < lhs.size(); ++i) validateMultiply(lhs[i], rhs[i]);
        const auto ctx = lhs[0].context;
        const size_t in_words = 2 * lhs[0].polyWords(), out_words = 3 * lhs[0].polyWords();
        std::vector<uint64_t> a(in_words * lhs.size()), b(in_words * lhs.size()), o(out_words * lhs.size());
        for (size_t i = 0; i < lhs.size(); ++i) {
            std::copy(lhs[i].data.begin(), lhs[i].data.end(), a.begin() + i * in_words);
            std::copy(rhs[i].data.begin(), rhs[i].data.end(), b.begin() + i * in_words);
        }
        check(hecuda_bfv_multiply(ctx->handle(), a.data(), b.data(), o.data(), (int64_t)lhs.size()));
        for (size_t i = 0; i < lhs.size(); ++i) {
            lhs[i].polyCount = 3;
            lhs[i].data.assign(o.begin() + i * out_words, o.begin() + (i + 1) * out_words);
        }
    }

    // Bfv.relinearize (Bfv.swift:201-219): 3 polys -> 2 polys
    static void relinearize(Ciphertext &ct, const EvaluationKey &key) {
        if (ct.correctionFactor != 1) throw HeError(HeError::invalidCiphertext, "correction factor must be 1");
        if (ct.polyCount != 3) throw HeError(HeError::invalidCiphertext, "ciphertext must have three polys when relinearizing");
        if (!(*ct.context == *key.context)) throw HeError(HeError::invalidContext, "key belongs to another context");
        Ciphertext out(ct.context, 2, ct.moduliCount);
        check(hecuda_bfv_relinearize(ct.context->handle(), key.handle(), ct.data.data(), ct.moduliCount, out.data.data(), 1));
        ct = std::move(out);
    }

    // Bfv.modSwitchDown (Bfv.swift:163-171): drops the last modulus of every poly
    static void modSwitchDown(Ciphertext &ct) {
        if (ct.correctionFactor != 1) throw HeError(HeError::invalidCiphertext, "correction factor must be 1");
        if (ct.moduliCount < 2) throw HeError(HeError::invalidPolyContext, "no next context");  // PolyRq.swift:366-368
        Ciphertext out(ct.context, ct.polyCount, ct.moduliCount - 1);
        check(hecuda_bfv_mod_switch_down(ct.context->handle(), ct.data.data(), ct.polyCount, ct.moduliCount, out.data.data(), 1));
        ct = std::move(out);
    }

    // mulAssign + relinearize (+ modSwitchDown when modSwitch) for a whole batch in one device pass -- the sequence
    // the reference's callers run back to back (RlweBenchmark.swift:387-493, PirUtil.swift:447-480).  The 3-poly
    // product stays on the device; results equal the three separate calls.
    static void mulRelinearizeAssign(std::vector<Ciphertext> &lhs, const std::vector<Ciphertext> &rhs, const EvaluationKey &key,
                                     bool modSwitch = false) {
        if (lhs.size() != rhs.size()) throw HeError(HeError::incompatibleCiphertexts, "batch sizes differ");
        if (lhs.empty()) return;
        for (size_t i = 0; i < lhs.size(); ++i) validateMultiply(lhs[i], rhs[i]);
        const auto ctx = lhs[0].context;
        if (!(*ctx == *key.context)) throw HeError(HeError::invalidContext, "key belongs to another context");
        const int rows = lhs[0].moduliCount;
        if (modSwitch && rows < 2) throw HeError(HeError::invalidPolyContext, "no next context");
        const int outRows = modSwitch ? rows - 1 : rows;
        const size_t n = lhs[0].polyWords() / (size_t)rows;
        const size_t in_words = 2 * lhs[0].polyWords(), out_words = 2 * (size_t)outRows * n;
        std::vector<uint64_t> a(in_words * lhs.size()), b(in_words * lhs.size()), o(out_words * lhs.size());
        for (size_t i = 0; i < lhs.size(); ++i) {
            std::copy(lhs[i].data.begin(), lhs[i].data.end(), a.begin() + i * in_words);
            std::copy(rhs[i].data.begin(), rhs[i].data.end(), b.begin() + i * in_words);
        }
        check(hecuda_bfv_multiply_relinearize(ctx->handle(), key.handle(), a.data(), b.data(), modSwitch ? 1 : 0, o.data(),
                                              (int64_t)lhs.size()));
        for (size_t i = 0; i < lhs.size(); ++i) {
            lhs[i].moduliCount = outRows;
            lhs[i].data.assign(o.begin() + i * out_words, o.begin() + (i + 1) * out_words);
        }
    }

    // relinearize + modSwitchDown in one device pass (3 polys at `moduliCount` rows -> 2 polys at one row fewer)
    static void relinearizeModSwitchDown(Ciphertext &ct, const EvaluationKey &key) {
        if (ct.correctionFactor != 1) throw HeError(HeError::invalidCiphertext, "correction factor must be 1");
        if (ct.polyCount != 3) throw HeError(HeError::invalidCiphertext, "ciphertext must have three polys when relinearizing");
        if (!(*ct.context == *key.context)) throw HeError(HeError::invalidContext, "key belongs to another context");
        if (ct.moduliCount < 2) throw HeError(HeError::invalidPolyContext, "no next context");
        Ciphertext out(ct.context, 2, ct.moduliCount - 1);
        check(hecuda_bfv_relinearize_mod_switch_down(ct.context->handle(), key.handle(), ct.data.data(), ct.moduliCount,
                                                     out.data.data(), 1));
        ct = std::move(out);
    }

    // Bfv.modSwitchDownToSingle (HeScheme.swift:1481-1485)
    static void modSwitchDownToSingle(Ciphertext &ct) {
        while (ct.moduliCount > 1) modSwitchDown(ct);
    }

    // validateEquality for the coefficient-wise ciphertext operations (HeScheme.swift:1326-1340)
    static void validateSameShape(const Ciphertext &lhs, const Ciphertext &rhs) {
        if (!lhs.context || !rhs.context || !(*lhs.context == *rhs.context))
            throw HeError(HeError::invalidContext, "ciphertexts have different contexts");
        if (lhs.polyCount != rhs.polyCount || lhs.moduliCount != rhs.moduliCount || lhs.correctionFactor != rhs.correctionFactor)
            throw HeError(HeError::incompatibleCiphertexts, "ciphertexts have different shapes");
    }
    // Bfv.addAssign / subAssign / negAssign on canonical ciphertexts (Bfv.swift:61-125): coefficient-wise on the polys
    static void addAssign(Ciphertext &lhs, const Ciphertext &rhs) {
        validateSameShape(lhs, rhs);
        check(hecuda_poly_add(lhs.context->handle(), HECUDA_BASE_Q, lhs.data.data(), rhs.data.data(), lhs.moduliCount, lhs.polyCount));
    }
    static void subAssign(Ciphertext &lhs, const Ciphertext &rhs) {
        validateSameShape(lhs, rhs);
        check(hecuda_poly_sub(lhs.context->handle(), HECUDA_BASE_Q, lhs.data.data(), rhs.data.data(), lhs.moduliCount, lhs.polyCount));
    }
    static void negAssign(Ciphertext &ct) {
        check(hecuda_poly_neg(ct.context->handle(), HECUDA_BASE_Q, ct.data.data(), ct.moduliCount, ct.polyCount));
    }

    // Bfv.applyGalois (Bfv.swift:174-198); rotateColumns / swapRows (HeScheme.swift:1463-1478) are applyGalois with
    // GaloisElement.rotatingColumns / swappingRows (PolyRq/Galois.swift:174-212)
    static void applyGalois(Ciphertext &ct, uint32_t element, const EvaluationKey &key) {
        if (ct.correctionFactor != 1) throw HeError(HeError::invalidCiphertext, "correction factor must be 1");
        if (ct.polyCount != freshCiphertextPolyCount) throw HeError(HeError::invalidCiphertext, "ciphertext must have two polys");
        if (!(*ct.context == *key.context)) throw HeError(HeError::invalidContext, "key belongs to another context");
        Ciphertext out(ct.context, 2, ct.moduliCount);
        check(hecuda_bfv_apply_galois(ct.context->handle(), key.handle(), ct.data.data(), ct.moduliCount, element, out.data.data(), 1));
        ct = std::move(out);
    }
    static uint32_t rotatingColumnsElement(int step, int64_t degree) {
        uint64_t positive = (uint64_t)(step < 0 ? -step : step);
        if (positive == 0 || positive >= (uint64_t)(degree >> 1)) throw HeError(HeError::invalidCiphertext, "invalidRotationStep");
        if (step > 0) positive = (uint64_t)(degree >> 1) - positive;
        uint64_t g = 1, base = 3, mod = 2 * (uint64_t)degree;
        for (uint64_t e = positive; e; e >>= 1) {
            if (e & 1) g = g * base % mod;
            base = base * base % mod;
        }
        return (uint32_t)g;
    }
    static void rotateColumns(Ciphertext &ct, int step, const EvaluationKey &key) {
        applyGalois(ct, rotatingColumnsElement(step, ct.context->degree), key);
    }
    static void swapRows(Ciphertext &ct, const EvaluationKey &key) {
        applyGalois(ct, (uint32_t)(2 * ct.context->degree - 1), key);
    }

    // Bfv.innerProduct(ciphertexts:plaintexts:) (Bfv.swift:476-505): Eval ciphertexts x optional Eval plaintexts
    static Ciphertext innerProduct(const std::vector<Ciphertext> &ciphertexts, const std::vector<const PolyRq *> &plaintexts) {
        if (ciphertexts.empty()) throw HeError(HeError::invalidCiphertext, "Empty ciphertexts");
        if (ciphertexts.size() != plaintexts.size()) throw HeError(HeError::incompatibleCiphertexts, "counts differ");
        const Ciphertext &first = ciphertexts[0];
        const size_t ctWords = (size_t)first.polyCount * first.polyWords(), ptWords = first.polyWords();
        std::vector<uint64_t> cts(ctWords * ciphertexts.size()), pts(ptWords * ciphertexts.size(), 0);
        std::vector<uint8_t> present(ciphertexts.size(), 0);
        for (size_t k = 0; k < ciphertexts.size(); ++k) {
            if (ciphertexts[k].polyCount != first.polyCount || ciphertexts[k].moduliCount != first.moduliCount)
                throw HeError(HeError::incompatibleCiphertexts, "ciphertexts have different shapes");
            std::copy(ciphertexts[k].data.begin(), ciphertexts[k].data.end(), cts.begin() + k * ctWords);
            if (plaintexts[k]) {
                if (plaintexts[k]->moduliCount != first.moduliCount) throw HeError(HeError::invalidPolyContext, "plaintext moduli count");
                std::copy(plaintexts[k]->data.begin(), plaintexts[k]->data.end(), pts.begin() + k * ptWords);
                present[k] = 1;
            }
        }
        Ciphertext out(first.context, first.polyCount, first.moduliCount);
        check(hecuda_bfv_inner_product_plaintexts(first.context->handle(), cts.data(), first.polyCount, first.moduliCount,
                                                  (int64_t)ciphertexts.size(), pts.data(), present.data(), out.data.data(), 1));
        return out;
    }

    // ---- the plaintext side.  A Coeff plaintext is its N coefficients (< t); an Eval plaintext is a PolyRq.
    // Context.supportsSimdEncoding (Context.swift:63-65)
    static bool supportsSimdEncoding(const Context &context) {
        int32_t supported = 0;
        check(hecuda_context_supports_simd(context.handle(), &supported));
        return supported != 0;
    }
    // Bfv.encode(context:values:format: .simd) (Encoding.swift:197-235): up to N values < t -> Coeff plaintext
    static std::vector<uint64_t> encodeSimd(const Context &context, const std::vector<uint64_t> &values) {
        std::vector<uint64_t> out((size_t)context.degree);
        check(hecuda_bfv_encode_simd(context.handle(), values.data(), (int32_t)values.size(), 0, out.data(), 1));
        return out;
    }
    // Bfv.encode(context:values:format: .simd, moduliCount:) (Bfv+Encode.swift:45-50) -> Eval plaintext
    static PolyRq encodeSimd(const std::shared_ptr<const Context> &context, const std::vector<uint64_t> &values, int moduliCount) {
        PolyRq out(context, moduliCount);
        check(hecuda_bfv_encode_simd(context->handle(), values.data(), (int32_t)values.size(), moduliCount, out.data.data(), 1));
        return out;
    }
    // Bfv.decodeCoeff(plaintext:format: .simd) (Encoding.swift:237-245): N slot values
    static std::vector<uint64_t> decodeSimd(const Context &context, const std::vector<uint64_t> &plaintext) {
        if (plaintext.size() != (size_t)context.degree) throw HeError(HeError::invalidPolyContext, "plaintext must have N coefficients");
        std::vector<uint64_t> out((size_t)context.degree);
        check(hecuda_bfv_decode_simd(context.handle(), plaintext.data(), 0, out.data(), 1));
        return out;
    }
    // Bfv.decodeEval(plaintext:format: .simd) (Bfv+Encode.swift:76-80)
    static std::vector<uint64_t> decodeSimd(const PolyRq &plaintext) {
        std::vector<uint64_t> out((size_t)plaintext.context->degree);
        check(hecuda_bfv_decode_simd(plaintext.context->handle(), plaintext.data.data(), plaintext.moduliCount, out.data(), 1));
        return out;
    }
    // plaintextTranslate's guards (Bfv+Encrypt.swift:80-83)
    static void validateTranslate(const Ciphertext &ct, const std::vector<uint64_t> &plaintext) {
        if (ct.correctionFactor != 1) throw HeError(HeError::invalidCiphertext, "invalidCorrectionFactor: correction factor must be 1");
        if (plaintext.size() != (size_t)ct.context->degree) throw HeError(HeError::invalidPolyContext, "plaintext must have N coefficients");
    }
    static void translate(Ciphertext &ct, const std::vector<uint64_t> &plaintext, int32_t op) {
        validateTranslate(ct, plaintext);
        check(hecuda_bfv_plaintext_translate(ct.context->handle(), ct.data.data(), ct.polyCount, ct.moduliCount, plaintext.data(), 1,
                                             op, ct.data.data(), 1));
    }
    // Bfv.addAssignCoeff / subAssignCoeff (Bfv.swift:110-117): ciphertext +-= Coeff plaintext
    static void addAssignCoeff(Ciphertext &ct, const std::vector<uint64_t> &plaintext) { translate(ct, plaintext, HECUDA_PLAINTEXT_ADD); }
    static void subAssignCoeff(Ciphertext &ct, const std::vector<uint64_t> &plaintext) { translate(ct, plaintext, HECUDA_PLAINTEXT_SUB); }
    // HeScheme.subCoeff(plaintext, ciphertext) (HeScheme.swift:1540-1542): plaintext - ciphertext
    static Ciphertext subCoeff(const std::vector<uint64_t> &plaintext, const Ciphertext &ct) {
        Ciphertext out = ct;
        translate(out, plaintext, HECUDA_PLAINTEXT_SUB_FROM);
        return out;
    }

    // PolyRq.forwardNtt / inverseNtt (in place; the reference consumes `self` and returns the other format)
    static void forwardNtt(PolyRq &poly) {
        check(hecuda_ntt_forward(poly.context->handle(), HECUDA_BASE_Q, poly.data.data(), poly.moduliCount, 1));
    }
    static void inverseNtt(PolyRq &poly) {
        check(hecuda_ntt_inverse(poly.context->handle(), HECUDA_BASE_Q, poly.data.data(), poly.moduliCount, 1));
    }
};

}  // namespace he
