// oprf_client.cu -- the symmetric-PIR OPRF client on the device (OprfClient, SymmetricPir/SymmetricPirProtocol.swift:
// 62-133), one thread per query, for batches of queries:
//
//   blind_kernel    queryContext(at:) (:98-104), RFC 9497 Blind: query = Ser(r HashToGroup(input)) for the caller's r
//   verify_kernel   parse(oprfResponse:with:) (:106-117), first half: decode the query and the evaluated element, check
//                   the DLEQ proof (RFC 9497 2.2.2 VerifyProof over one element) and set the query's status
//   unblind_kernel  parse's second half, for the verified queries: N = r^-1 D and Finalize's SHA-384
//   open_kernel     decrypt(encryptedEntry:with:) (:119-132): AES.GCM.open with key h[24:48], nonce h[0:12], the last
//                   16 bytes as the tag; nothing unauthenticated is written
//
// The field, group and hashing arithmetic is in p384.cuh, AES-GCM in aes_gcm.cuh.  The server's public key is decoded
// and its composite seed hashed once per call on the host, and passed to the kernels by value.  The device copies of
// the blinds, the OPRF outputs and the opened values are zeroized before they are freed.
#include <algorithm>

#include "aes_gcm.cuh"
#include "capi_internal.hpp"
#include "oprf_host.hpp"
#include "p384.cuh"

using namespace hecuda;
using namespace hecuda::api;
using namespace hecuda::api::oprf_host;

namespace {

constexpr int kThreads = 128;
constexpr int kNonceBytes = 12, kAesKeyOffset = 24, kTagBytes = 16;
constexpr uint8_t kRejected = 1, kInvalidContext = 2;  // hecuda_oprf_finalize's statuses

__constant__ unsigned char c_sbox[256];
__constant__ drbg::u32w c_te0[256];

// The server's public key, decoded and hashed on the host: pkS (Jacobian, Montgomery), Ser(pkS) and the composite seed
struct ServerKey {
    p384::Point pk;
    unsigned char ser[p384::kElementBytes];
    unsigned char seed[p384::kSeedBytes];
};

__device__ __forceinline__ void load_scalar(p384::Fe &r, const unsigned char *__restrict__ be) {
    unsigned char b[p384::kScalarBytes];
    for (int j = 0; j < p384::kScalarBytes; ++j) b[j] = be[j];
    p384::from_bytes(r, b);
}

// queries first .. first + count: queries[i] = Ser(r_i HashToGroup(input_i)) and status 0, or 49 zero bytes and status
// 1 when r_i is not in [1, n - 1]
__global__ void __launch_bounds__(kThreads) blind_kernel(const unsigned char *__restrict__ inputs,
                                                        const uint64_t *__restrict__ offsets, long long first,
                                                        long long count, const unsigned char *__restrict__ blinds,
                                                        unsigned char *__restrict__ queries,
                                                        uint8_t *__restrict__ status) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    p384::Fe r;
    load_scalar(r, blinds + i * p384::kScalarBytes);
    unsigned char query[p384::kElementBytes] = {};
    const bool ok = p384::scalar_valid(r);
    if (ok) p384::blind(query, r, inputs + offsets[i], (long long)(offsets[i + 1] - offsets[i]));
    for (int j = 0; j < p384::kElementBytes; ++j) queries[i * p384::kElementBytes + j] = query[j];
    status[i] = ok ? 0 : 1;
}

// queries first .. first + count: status 2 for a blind outside [1, n - 1] or an invalid query encoding, 1 for an
// invalid evaluated element or a proof that does not verify, 0 otherwise
__global__ void __launch_bounds__(kThreads) verify_kernel(const ServerKey key, const unsigned char *__restrict__ blinds,
                                                         const unsigned char *__restrict__ queries,
                                                         const unsigned char *__restrict__ responses, long long first,
                                                         long long count, uint8_t *__restrict__ status) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    p384::Fe r;
    load_scalar(r, blinds + i * p384::kScalarBytes);
    unsigned char blinded[p384::kElementBytes], response[p384::kResponseBytes];
    for (int j = 0; j < p384::kElementBytes; ++j) blinded[j] = queries[i * p384::kElementBytes + j];
    for (int j = 0; j < p384::kResponseBytes; ++j) response[j] = responses[i * p384::kResponseBytes + j];
    p384::Point b, d;
    uint8_t s = 0;
    if (!p384::scalar_valid(r) || !p384::decompress(b, blinded)) {
        s = kInvalidContext;
    } else if (!p384::decompress(d, response) ||
               !p384::verify_proof(key.pk, key.ser, key.seed, b, blinded, d, response,
                                   response + p384::kElementBytes)) {
        s = kRejected;
    }
    status[i] = s;
}

// queries first .. first + count: outputs[i] = Finalize's hash for status 0, else 48 zero bytes
__global__ void __launch_bounds__(kThreads) unblind_kernel(const unsigned char *__restrict__ inputs,
                                                          const uint64_t *__restrict__ offsets,
                                                          const unsigned char *__restrict__ blinds,
                                                          const unsigned char *__restrict__ responses, long long first,
                                                          long long count, const uint8_t *__restrict__ status,
                                                          unsigned char *__restrict__ outputs) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    unsigned char h[p384::kOutputBytes] = {};
    if (status[i] == 0) {
        p384::Fe r;
        load_scalar(r, blinds + i * p384::kScalarBytes);
        unsigned char evaluated[p384::kElementBytes];
        for (int j = 0; j < p384::kElementBytes; ++j) evaluated[j] = responses[i * p384::kResponseBytes + j];
        p384::Point d;
        p384::decompress(d, evaluated);  // verify_kernel decoded it
        p384::unblind_finalize(h, r, d, inputs + offsets[i], (long long)(offsets[i + 1] - offsets[i]));
    }
    for (int j = 0; j < p384::kOutputBytes; ++j) outputs[i * p384::kOutputBytes + j] = h[j];
}

// entries first .. first + count: values[off_i : off_{i+1} - 16] = the plaintext and the 16 bytes after it zero,
// status 0; or values[off_i : off_{i+1}] all zero and status 1 when the tag does not match or the entry is shorter
// than a tag
__global__ void __launch_bounds__(kThreads) open_kernel(const unsigned char *__restrict__ oprf,
                                                       const unsigned char *__restrict__ sealed,
                                                       const uint64_t *__restrict__ offsets, long long first,
                                                       long long count, unsigned char *__restrict__ values,
                                                       uint8_t *__restrict__ status) {
    __shared__ unsigned char sbox[256];
    __shared__ drbg::u32w te0[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sbox[i] = c_sbox[i], te0[i] = c_te0[i];
    __syncthreads();
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= count) return;
    const long long i = first + t;
    const uint64_t at = offsets[i];
    const long long len = (long long)(offsets[i + 1] - at);
    bool ok = false;
    long long plain = 0;
    if (len >= kTagBytes) {
        const unsigned char *h = oprf + i * p384::kOutputBytes;
        drbg::u32w key[6], rk[gcm::kRoundKeyWords192];
        for (int w = 0; w < 6; ++w) {
            const unsigned char *q = h + kAesKeyOffset + 4 * w;
            key[w] = ((drbg::u32w)q[0] << 24) | ((drbg::u32w)q[1] << 16) | ((drbg::u32w)q[2] << 8) | q[3];
        }
        gcm::expand_key_192(key, rk, sbox);
        unsigned char nonce[kNonceBytes], tag[kTagBytes];
        for (int j = 0; j < kNonceBytes; ++j) nonce[j] = h[j];
        plain = len - kTagBytes;
        for (int j = 0; j < kTagBytes; ++j) tag[j] = sealed[at + plain + j];
        ok = gcm::open(rk, te0, sbox, nonce, sealed + at, plain, tag, values + at);
    }
    for (long long j = plain; j < len; ++j) values[at + j] = 0;
    status[i] = ok ? 0 : 1;
}

unsigned grid_for(long long items) { return (unsigned)((items + kThreads - 1) / kThreads); }

cudaError_t upload_aes_tables() {
    unsigned char sbox[256];
    drbg::u32w te0[256];
    drbg::make_tables(sbox, te0);
    cudaError_t e = cudaMemcpyToSymbol(c_sbox, sbox, sizeof(sbox));
    return e == cudaSuccess ? cudaMemcpyToSymbol(c_te0, te0, sizeof(te0)) : e;
}

// Device buffers of one call; the blinds, the OPRF outputs and the opened values are zeroized before they are freed.
struct Buffers {
    unsigned char *inputs = nullptr, *blinds = nullptr, *queries = nullptr, *responses = nullptr, *oprf = nullptr;
    unsigned char *sealed = nullptr, *values = nullptr;
    uint64_t *offsets = nullptr;
    uint8_t *status = nullptr;
    size_t blind_bytes = 0, oprf_bytes = 0, value_bytes = 0;
    ~Buffers() {
        if (blinds) cudaMemset(blinds, 0, std::max<size_t>(blind_bytes, 1));
        if (oprf) cudaMemset(oprf, 0, std::max<size_t>(oprf_bytes, 1));
        if (values) cudaMemset(values, 0, std::max<size_t>(value_bytes, 1));
        cudaDeviceSynchronize();
        for (void *p : {(void *)inputs, (void *)blinds, (void *)queries, (void *)responses, (void *)oprf, (void *)sealed,
                        (void *)values, (void *)offsets, (void *)status})
            cudaFree(p);
    }
};

// The OPRF inputs and the blinds on the device
cudaError_t upload_queries(Buffers &b, const uint8_t *inputs, const uint64_t *offsets, int64_t count,
                           const uint8_t *blinds) {
    b.blind_bytes = (size_t)count * p384::kScalarBytes;
    cudaError_t e = upload_new(&b.inputs, inputs, (size_t)offsets[count]);
    if (e == cudaSuccess) e = upload_new(&b.offsets, offsets, (size_t)(count + 1) * sizeof(uint64_t));
    if (e == cudaSuccess) e = upload_new(&b.blinds, blinds, b.blind_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&b.status, (size_t)count);
    return e;
}

// OprfPublicKey(compressedRepresentation:): a valid SEC1-compressed point, then Ser(pkS) and the composite seed
int32_t decode_server_key(const uint8_t *public_key, ServerKey &key) {
    if (!p384::decompress(key.pk, public_key))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid OPRF public key: not a SEC1-compressed P-384 point");
    std::copy(public_key, public_key + p384::kElementBytes, key.ser);  // a valid encoding is unique
    p384::composite_seed(key.seed, key.ser);
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_oprf_blind(const uint8_t *inputs, const uint64_t *offsets, int64_t count, const uint8_t *blinds,
                          uint8_t *queries, uint8_t *status) {
    if (!blinds || !queries || !status) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_inputs(inputs, offsets, count, "OPRF input");
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) return rc;
    const size_t query_bytes = (size_t)count * p384::kElementBytes;
    cudaError_t e;
    {
        Buffers b;
        e = upload_queries(b, inputs, offsets, count, blinds);
        if (e == cudaSuccess) e = cudaMalloc(&b.queries, query_bytes);
        if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
            return launch(blind_kernel, grid_for(part), kThreads, 0, 0, (const unsigned char *)b.inputs,
                          (const uint64_t *)b.offsets, (long long)first, (long long)part,
                          (const unsigned char *)b.blinds, b.queries, b.status);
        });
        if (e == cudaSuccess) e = cudaMemcpy(queries, b.queries, query_bytes, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(status, b.status, (size_t)count, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "OPRF blind");
}

int32_t hecuda_oprf_finalize(const uint8_t *public_key, const uint8_t *inputs, const uint64_t *offsets, int64_t count,
                             const uint8_t *blinds, const uint8_t *queries, const uint8_t *responses, uint8_t *outputs,
                             uint8_t *status) {
    if (!public_key || !blinds || !queries || !responses || !outputs || !status)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = check_inputs(inputs, offsets, count, "OPRF input");
    ServerKey key;
    if (!rc) rc = decode_server_key(public_key, key);
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) return rc;
    const size_t response_bytes = (size_t)count * p384::kResponseBytes;
    cudaError_t e;
    {
        Buffers b;
        b.oprf_bytes = (size_t)count * p384::kOutputBytes;
        e = upload_queries(b, inputs, offsets, count, blinds);
        if (e == cudaSuccess) e = upload_new(&b.queries, queries, (size_t)count * p384::kElementBytes);
        if (e == cudaSuccess) e = upload_new(&b.responses, responses, response_bytes);
        if (e == cudaSuccess) e = cudaMalloc(&b.oprf, b.oprf_bytes);
        if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
            return launch(verify_kernel, grid_for(part), kThreads, 0, 0, key, (const unsigned char *)b.blinds,
                          (const unsigned char *)b.queries, (const unsigned char *)b.responses, (long long)first,
                          (long long)part, b.status);
        });
        if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
            return launch(unblind_kernel, grid_for(part), kThreads, 0, 0, (const unsigned char *)b.inputs,
                          (const uint64_t *)b.offsets, (const unsigned char *)b.blinds,
                          (const unsigned char *)b.responses, (long long)first, (long long)part,
                          (const uint8_t *)b.status, b.oprf);
        });
        if (e == cudaSuccess) e = cudaMemcpy(outputs, b.oprf, b.oprf_bytes, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(status, b.status, (size_t)count, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "OPRF finalize");
}

int32_t hecuda_symmetric_pir_open(const uint8_t *oprf_outputs, const uint8_t *sealed, const uint64_t *sealed_offsets,
                                  int64_t count, uint8_t *values, uint8_t *status) {
    if (!oprf_outputs || !sealed || !sealed_offsets || !values || !status || count < 0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    uint64_t longest = 0;
    int32_t rc = check_rows(sealed_offsets, count, "sealed entry", longest);
    if (!rc && count > 0) rc = have_device();
    if (rc || count == 0) return rc;
    cudaError_t e;
    {
        Buffers b;
        b.oprf_bytes = (size_t)count * p384::kOutputBytes;
        b.value_bytes = (size_t)sealed_offsets[count];
        e = upload_aes_tables();
        if (e == cudaSuccess) e = upload_new(&b.oprf, oprf_outputs, b.oprf_bytes);
        if (e == cudaSuccess) e = upload_new(&b.sealed, sealed, b.value_bytes);
        if (e == cudaSuccess) e = upload_new(&b.offsets, sealed_offsets, (size_t)(count + 1) * sizeof(uint64_t));
        if (e == cudaSuccess) e = cudaMalloc(&b.values, std::max<size_t>(b.value_bytes, 1));
        if (e == cudaSuccess) e = cudaMemset(b.values, 0, std::max<size_t>(b.value_bytes, 1));  // bytes before offsets[0]
        if (e == cudaSuccess) e = cudaMalloc(&b.status, (size_t)count);
        if (e == cudaSuccess) e = for_each_part(count, [&](int64_t first, int64_t part) {
            return launch(open_kernel, grid_for(part), kThreads, 0, 0, (const unsigned char *)b.oprf,
                          (const unsigned char *)b.sealed, (const uint64_t *)b.offsets, (long long)first,
                          (long long)part, b.values, b.status);
        });
        if (e == cudaSuccess && b.value_bytes) e = cudaMemcpy(values, b.values, b.value_bytes, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(status, b.status, (size_t)count, cudaMemcpyDeviceToHost);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "symmetric PIR open");
}

}  // extern "C"
