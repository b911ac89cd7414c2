// symmetric_pir.cu -- symmetric keyword PIR's per-row processing on the device (SymmetricPir/SymmetricPirDatabase.swift:
// 186-211, config OPRF_P384_AES_GCM_192_NONCE_96_TAG_128):
//
//   oprf_evaluate_kernel   h = RFC 9497 Evaluate(k, keyword) over P384-SHA384 for every row, one thread each
//   seal_kernel            keyword' = h[0:16] and value' = AES-GCM-192-seal(key h[24:48], nonce h[0:12], value), one
//                          thread each
//   public_key_kernel      k G, compressed (SymmetricPirConfig.clientConfig().serverPublicKey)
//
// and the online OPRF server (OprfServer.computeResponse, SymmetricPir/SymmetricPirProtocol.swift:39-59), RFC 9497
// BlindEvaluate with the DLEQ proof, one thread per query:
//
//   proof_setup_kernel     bm = Ser(k G) and ComputeCompositesFast's seed, once per call
//   blind_evaluate_kernel  decode B, Ser(k B) into the response, the composite M = d0 B staged for the next kernel
//   proof_kernel           the nonce r, Z = k M, t2 = r G, t3 = r M, the challenge c and s = r - c k into the response
//
// The field, group and hash-to-curve arithmetic is in p384.cuh, SHA-384 in sha512.cuh, AES-GCM in aes_gcm.cuh.  The key
// is checked and recoded on the host once; its recoding, its plain copy (the server's s = r - c k) and every row's h
// (which holds the row's AES key) live in device buffers that are zeroized before they are freed.  r never leaves the
// thread that derives it.
#include <algorithm>
#include <cstring>
#include <string>

#include "aes_gcm.cuh"
#include "capi_internal.hpp"
#include "oprf_host.hpp"
#include "p384.cuh"

using namespace hecuda;
using namespace hecuda::api;
using namespace hecuda::api::oprf_host;

namespace {

constexpr int kThreads = 128;
constexpr int kRecodingBytes = p384::kDigits + 1;  // 96 digits, then the flip flag
constexpr int kKeywordBytes = 16, kNonceBytes = 12, kAesKeyOffset = 24, kTagBytes = 16;

__constant__ unsigned char c_sbox[256];
__constant__ drbg::u32w c_te0[256];

// the recoding into shared memory; every thread of the block reads it
__device__ __forceinline__ void stage_recoding(signed char *s, const signed char *__restrict__ recoding) {
    for (int i = threadIdx.x; i < kRecodingBytes; i += blockDim.x) s[i] = recoding[i];
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) public_key_kernel(const signed char *__restrict__ recoding,
                                                             unsigned char *__restrict__ out) {
    __shared__ signed char digits[kRecodingBytes];
    stage_recoding(digits, recoding);
    if (threadIdx.x != 0) return;
    p384::Point g, r;
    p384::generator(g);
    p384::scalar_mul(r, g, digits);
    p384::compress(out, r);
}

// rows first .. first + count of the ragged inputs -> out[row][48]
__global__ void __launch_bounds__(kThreads) oprf_evaluate_kernel(const unsigned char *__restrict__ inputs,
                                                                const uint64_t *__restrict__ offsets, long long first,
                                                                long long count, const signed char *__restrict__ recoding,
                                                                unsigned char *__restrict__ out) {
    __shared__ signed char digits[kRecodingBytes];
    stage_recoding(digits, recoding);
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    unsigned char h[p384::kOutputBytes];
    p384::oprf_evaluate(h, digits, inputs + offsets[i], (long long)(offsets[i + 1] - offsets[i]));
    for (int j = 0; j < p384::kOutputBytes; ++j) out[i * p384::kOutputBytes + j] = h[j];
}

// rows first .. first + count: keyword' and ciphertext || tag, row i's value at value_offsets[i] + 16 i
__global__ void __launch_bounds__(kThreads) seal_kernel(const unsigned char *__restrict__ oprf,
                                                       const unsigned char *__restrict__ values,
                                                       const uint64_t *__restrict__ value_offsets, long long first,
                                                       long long count, unsigned char *__restrict__ keywords_out,
                                                       unsigned char *__restrict__ values_out) {
    __shared__ unsigned char sbox[256];
    __shared__ drbg::u32w te0[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sbox[i] = c_sbox[i], te0[i] = c_te0[i];
    __syncthreads();
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    const unsigned char *h = oprf + i * p384::kOutputBytes;
    for (int j = 0; j < kKeywordBytes; ++j) keywords_out[i * kKeywordBytes + j] = h[j];
    drbg::u32w key[6], rk[gcm::kRoundKeyWords192];
    for (int w = 0; w < 6; ++w) {
        const unsigned char *q = h + kAesKeyOffset + 4 * w;
        key[w] = ((drbg::u32w)q[0] << 24) | ((drbg::u32w)q[1] << 16) | ((drbg::u32w)q[2] << 8) | q[3];
    }
    gcm::expand_key_192(key, rk, sbox);
    unsigned char nonce[kNonceBytes];
    for (int j = 0; j < kNonceBytes; ++j) nonce[j] = h[j];
    const uint64_t at = value_offsets[i];
    gcm::seal(rk, te0, sbox, nonce, values + at, (long long)(value_offsets[i + 1] - at), values_out + at + kTagBytes * i);
}

// setup = bm (49 bytes) || seed (48 bytes)
constexpr int kSetupBytes = p384::kElementBytes + p384::kSeedBytes;

__global__ void __launch_bounds__(kThreads) proof_setup_kernel(const signed char *__restrict__ recoding,
                                                              unsigned char *__restrict__ setup) {
    __shared__ signed char digits[kRecodingBytes];
    stage_recoding(digits, recoding);
    if (threadIdx.x != 0) return;
    p384::Point g, r;
    p384::generator(g);
    p384::scalar_mul(r, g, digits);
    p384::compress(setup, r);
    p384::composite_seed(setup + p384::kElementBytes, setup);
}

// queries first .. first + count: responses[i][0:49] = Ser(k B_i) and staged[2i], staged[2i + 1] = M_i, or status 1
// and 145 zero bytes for an invalid query
__global__ void __launch_bounds__(kThreads) blind_evaluate_kernel(const unsigned char *__restrict__ queries,
                                                                 long long first, long long count,
                                                                 const signed char *__restrict__ recoding,
                                                                 const unsigned char *__restrict__ setup,
                                                                 unsigned char *__restrict__ responses,
                                                                 uint8_t *__restrict__ status,
                                                                 p384::Fe *__restrict__ staged) {
    __shared__ signed char digits[kRecodingBytes];
    stage_recoding(digits, recoding);
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    unsigned char query[p384::kElementBytes], evaluated[p384::kElementBytes] = {};
    for (int j = 0; j < p384::kElementBytes; ++j) query[j] = queries[i * p384::kElementBytes + j];
    p384::Fe mx = {}, my = {};
    const bool ok = p384::blind_evaluate_composite(evaluated, mx, my, query, digits, setup + p384::kElementBytes);
    unsigned char *out = responses + i * p384::kResponseBytes;
    for (int j = 0; j < p384::kElementBytes; ++j) out[j] = ok ? evaluated[j] : 0;
    for (int j = p384::kElementBytes; j < p384::kResponseBytes; ++j) out[j] = 0;
    status[i] = ok ? 0 : 1;
    staged[2 * i] = mx, staged[2 * i + 1] = my;
}

// queries first .. first + count with status 0: responses[i][49:145] = c || s.  r = 0 (negligible) marks the query
// invalid like a bad encoding.
__global__ void __launch_bounds__(kThreads) proof_kernel(const unsigned char *__restrict__ queries, long long first,
                                                        long long count, const signed char *__restrict__ recoding,
                                                        const p384::Fe *__restrict__ secret,
                                                        const unsigned char *__restrict__ setup,
                                                        const unsigned char *__restrict__ seed32,
                                                        const p384::Fe *__restrict__ staged,
                                                        unsigned char *__restrict__ responses,
                                                        uint8_t *__restrict__ status) {
    __shared__ signed char digits[kRecodingBytes];
    stage_recoding(digits, recoding);
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    if (status[i]) return;
    unsigned char query[p384::kElementBytes], seed[p384::kNonceSeedBytes];
    for (int j = 0; j < p384::kElementBytes; ++j) query[j] = queries[i * p384::kElementBytes + j];
    for (int j = 0; j < p384::kNonceSeedBytes; ++j) seed[j] = seed32[j];
    const p384::Fe k = *secret;
    p384::Fe r;
    p384::proof_nonce(r, k, seed, query);
    unsigned char *out = responses + i * p384::kResponseBytes;
    if (p384::is_zero(r)) {
        for (int j = 0; j < p384::kElementBytes; ++j) out[j] = 0;
        status[i] = 1;
        return;
    }
    unsigned char proof[p384::kProofBytes];
    p384::generate_proof(proof, digits, k, setup, staged[2 * i], staged[2 * i + 1], r);
    for (int j = 0; j < p384::kProofBytes; ++j) out[p384::kElementBytes + j] = proof[j];
}

unsigned grid_for(long long items) { return (unsigned)((items + kThreads - 1) / kThreads); }

// Every launcher takes rows in parts of at most kMaxGridYZ, like the library's other batched launchers.
cudaError_t launch_oprf_evaluate(const unsigned char *d_inputs, const uint64_t *d_offsets, int64_t count,
                                 const signed char *d_recoding, unsigned char *d_out) {
    return for_each_part(count, [&](int64_t first, int64_t part) {
        return launch(oprf_evaluate_kernel, grid_for(part), kThreads, 0, 0, d_inputs, d_offsets, (long long)first,
                      (long long)part, d_recoding, d_out);
    });
}

cudaError_t launch_seal(const unsigned char *d_oprf, const unsigned char *d_values, const uint64_t *d_value_offsets,
                        int64_t count, unsigned char *d_keywords_out, unsigned char *d_values_out) {
    return for_each_part(count, [&](int64_t first, int64_t part) {
        return launch(seal_kernel, grid_for(part), kThreads, 0, 0, d_oprf, d_values, d_value_offsets, (long long)first,
                      (long long)part, d_keywords_out, d_values_out);
    });
}

cudaError_t launch_blind_evaluate(const unsigned char *d_queries, int64_t count, const signed char *d_recoding,
                                  const p384::Fe *d_secret, unsigned char *d_setup, const unsigned char *d_seed32,
                                  p384::Fe *d_staged, unsigned char *d_responses, uint8_t *d_status) {
    cudaError_t e = launch(proof_setup_kernel, 1, kThreads, 0, 0, d_recoding, d_setup);
    if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
        return launch(blind_evaluate_kernel, grid_for(part), kThreads, 0, 0, d_queries, (long long)first, (long long)part,
                      d_recoding, d_setup, d_responses, d_status, d_staged);
    });
    if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
        return launch(proof_kernel, grid_for(part), kThreads, 0, 0, d_queries, (long long)first, (long long)part,
                      d_recoding, d_secret, d_setup, d_seed32, (const p384::Fe *)d_staged, d_responses, d_status);
    });
    return e;
}

cudaError_t upload_aes_tables() {
    unsigned char sbox[256];
    drbg::u32w te0[256];
    drbg::make_tables(sbox, te0);
    cudaError_t e = cudaMemcpyToSymbol(c_sbox, sbox, sizeof(sbox));
    return e == cudaSuccess ? cudaMemcpyToSymbol(c_te0, te0, sizeof(te0)) : e;
}

// The key as OprfPrivateKey(rawRepresentation:) takes it: 48 big-endian bytes, 0 < k < n; recoded into `recoding`
int32_t recode_key(const uint8_t *secret_key, signed char recoding[kRecodingBytes]) {
    if (!secret_key) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null OPRF secret key");
    p384::Fe k;
    p384::from_bytes(k, secret_key);
    const bool valid = p384::scalar_valid(k);
    if (valid) p384::recode_scalar(k, recoding);
    wipe(&k, sizeof(k));
    return valid ? HECUDA_OK : fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid OPRF secret key: not in [1, n - 1] for P-384");
}

// Device buffers of one call; the key's recoding and plain copy and the OPRF outputs are zeroized before they are freed.
struct Buffers {
    signed char *recoding = nullptr;
    p384::Fe *secret = nullptr, *staged = nullptr;
    unsigned char *inputs = nullptr, *oprf = nullptr, *values = nullptr, *keywords_out = nullptr, *values_out = nullptr;
    unsigned char *setup = nullptr, *seed32 = nullptr;
    uint8_t *status = nullptr;
    uint64_t *offsets = nullptr, *value_offsets = nullptr;
    size_t oprf_bytes = 0;
    ~Buffers() {
        if (recoding) cudaMemset(recoding, 0, kRecodingBytes);
        if (secret) cudaMemset(secret, 0, sizeof(p384::Fe));
        if (oprf) cudaMemset(oprf, 0, std::max<size_t>(oprf_bytes, 1));
        cudaDeviceSynchronize();
        for (void *p : {(void *)recoding, (void *)secret, (void *)staged, (void *)inputs, (void *)oprf, (void *)values,
                        (void *)keywords_out, (void *)values_out, (void *)setup, (void *)seed32, (void *)status,
                        (void *)offsets, (void *)value_offsets})
            cudaFree(p);
    }
};

// Uploads the recoding and the inputs and runs the OPRF kernel: b.oprf holds count x 48 bytes
cudaError_t evaluate_on_device(Buffers &b, const signed char *recoding, const uint8_t *inputs, const uint64_t *offsets,
                               int64_t count) {
    b.oprf_bytes = (size_t)count * p384::kOutputBytes;
    cudaError_t e = upload_new(&b.recoding, recoding, kRecodingBytes);
    if (e == cudaSuccess) e = upload_new(&b.inputs, inputs, (size_t)offsets[count]);
    if (e == cudaSuccess) e = upload_new(&b.offsets, offsets, (size_t)(count + 1) * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&b.oprf, std::max<size_t>(b.oprf_bytes, 1));
    if (e == cudaSuccess) e = launch_oprf_evaluate(b.inputs, b.offsets, count, b.recoding, b.oprf);
    return e;
}

}  // namespace

extern "C" {

int32_t hecuda_oprf_public_key(const uint8_t *secret_key, uint8_t *public_key) {
    if (!public_key) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    signed char recoding[kRecodingBytes];
    int32_t rc = recode_key(secret_key, recoding);
    if (!rc) rc = have_device();
    if (rc) {
        wipe(recoding, sizeof(recoding));
        return rc;
    }
    cudaError_t e;
    {
        Buffers b;
        e = upload_new(&b.recoding, recoding, kRecodingBytes);
        wipe(recoding, sizeof(recoding));
        if (e == cudaSuccess) e = cudaMalloc(&b.values_out, HECUDA_OPRF_ELEMENT_BYTES);
        if (e == cudaSuccess) e = launch(public_key_kernel, 1, kThreads, 0, 0, (const signed char *)b.recoding, b.values_out);
        if (e == cudaSuccess) e = cudaMemcpy(public_key, b.values_out, HECUDA_OPRF_ELEMENT_BYTES, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "OPRF public key");
}

int32_t hecuda_oprf_evaluate(const uint8_t *secret_key, const uint8_t *inputs, const uint64_t *offsets, int64_t count,
                             uint8_t *outputs) {
    if (!outputs) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_inputs(inputs, offsets, count, "OPRF input");
    signed char recoding[kRecodingBytes];
    if (!rc) rc = recode_key(secret_key, recoding);
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) {
        wipe(recoding, sizeof(recoding));
        return rc;
    }
    cudaError_t e;
    {
        Buffers b;
        e = evaluate_on_device(b, recoding, inputs, offsets, count);
        wipe(recoding, sizeof(recoding));
        if (e == cudaSuccess) e = cudaMemcpy(outputs, b.oprf, b.oprf_bytes, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "OPRF evaluate");
}

int32_t hecuda_symmetric_pir_process(const uint8_t *secret_key, const uint8_t *keywords, const uint64_t *keyword_offsets,
                                     const uint8_t *values, const uint64_t *value_offsets, int64_t count,
                                     uint8_t *keywords_out, uint8_t *values_out) {
    if (!values || !value_offsets || !keywords_out || !values_out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_inputs(keywords, keyword_offsets, count, "OPRF input");  // the keywords
    uint64_t longest_value = 0;
    if (!rc) rc = check_rows(value_offsets, count, "value", longest_value);
    signed char recoding[kRecodingBytes];
    if (!rc) rc = recode_key(secret_key, recoding);
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) {
        wipe(recoding, sizeof(recoding));
        return rc;
    }
    const size_t value_bytes = (size_t)value_offsets[count];
    const size_t out_bytes = value_bytes + (size_t)kTagBytes * count;
    cudaError_t e;
    {
        Buffers b;
        e = evaluate_on_device(b, recoding, keywords, keyword_offsets, count);
        wipe(recoding, sizeof(recoding));
        if (e == cudaSuccess) e = upload_aes_tables();
        if (e == cudaSuccess) e = upload_new(&b.values, values, value_bytes);
        if (e == cudaSuccess) e = upload_new(&b.value_offsets, value_offsets, (size_t)(count + 1) * sizeof(uint64_t));
        if (e == cudaSuccess) e = cudaMalloc(&b.keywords_out, (size_t)kKeywordBytes * count);
        if (e == cudaSuccess) e = cudaMalloc(&b.values_out, std::max<size_t>(out_bytes, 1));
        if (e == cudaSuccess) e = launch_seal(b.oprf, b.values, b.value_offsets, count, b.keywords_out, b.values_out);
        if (e == cudaSuccess) e = cudaMemcpy(keywords_out, b.keywords_out, (size_t)kKeywordBytes * count, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(values_out, b.values_out, out_bytes, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "symmetric PIR process");
}

int32_t hecuda_oprf_blind_evaluate(const uint8_t *secret_key, const uint8_t *blinded_elements, int64_t count,
                                   const uint8_t *seed, uint8_t *responses, uint8_t *status) {
    if (!blinded_elements || !seed || !responses || !status || count < 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    signed char recoding[kRecodingBytes];
    int32_t rc = recode_key(secret_key, recoding);
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) {
        wipe(recoding, sizeof(recoding));
        return rc;
    }
    p384::Fe k;
    p384::from_bytes(k, secret_key);
    const size_t query_bytes = (size_t)count * p384::kElementBytes, response_bytes = (size_t)count * p384::kResponseBytes;
    cudaError_t e;
    {
        Buffers b;
        e = upload_new(&b.recoding, recoding, kRecodingBytes);
        if (e == cudaSuccess) e = upload_new(&b.secret, &k, sizeof(k));
        wipe(recoding, sizeof(recoding));
        wipe(&k, sizeof(k));
        if (e == cudaSuccess) e = upload_new(&b.seed32, seed, p384::kNonceSeedBytes);
        if (e == cudaSuccess) e = upload_new(&b.inputs, blinded_elements, query_bytes);
        if (e == cudaSuccess) e = cudaMalloc(&b.setup, kSetupBytes);
        if (e == cudaSuccess) e = cudaMalloc(&b.staged, (size_t)count * 2 * sizeof(p384::Fe));
        if (e == cudaSuccess) e = cudaMalloc(&b.values_out, response_bytes);
        if (e == cudaSuccess) e = cudaMalloc(&b.status, (size_t)count);
        if (e == cudaSuccess)
            e = launch_blind_evaluate(b.inputs, count, b.recoding, b.secret, b.setup, b.seed32, b.staged, b.values_out,
                                      b.status);
        if (e == cudaSuccess) e = cudaMemcpy(responses, b.values_out, response_bytes, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(status, b.status, (size_t)count, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "OPRF blind evaluate");
}

}  // extern "C"
