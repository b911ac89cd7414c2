// pnns_client.cu -- the PNNS client on the device: float vectors to encrypted .denseRow query matrices, and
// .denseColumn replies back to float distances, composed across several plaintext moduli (plaintext CRT).
//
//   Array2d.normalizedScaledAndRounded     PrivateNearestNeighborSearch/Util.swift:74-89
//   Client.generateQuery                   PrivateNearestNeighborSearch/Client.swift:73-91
//   PlaintextMatrix.denseRowPlaintexts     PrivateNearestNeighborSearch/PlaintextMatrix.swift:341-413
//   Client.decrypt                         Client.swift:99-127 (unpackDenseColumn PlaintextMatrix.swift:515-555,
//                                          CrtComposer.compose HomomorphicEncryption/CrtComposer.swift:76-97)
//
// The float arithmetic and the index maps are the __host__ __device__ helpers of process_db.cuh, which
// tests/emu/pnns_client_emulate.cu replays on the CPU.  A query is normalised, scattered into SIMD slots, encoded and
// encrypted without leaving the device; distances are decrypted, decoded and composed the same way.
#include <algorithm>
#include <cmath>
#include <vector>

#include "capi_internal.hpp"
#include "hostmath.hpp"

using namespace hecuda;
using namespace hecuda::api;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxPlaintextModuli = 8;  // PnnsCrt's capacity

// one thread per row: the sum of squares runs left to right, as the reference's reduce(0, +) does
__global__ void __launch_bounds__(kThreads) row_norm_kernel(const float *__restrict__ v, long long rows, long long cols,
                                                           float *__restrict__ norms) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    norms[r] = procdb::pnns_row_norm(v + r * cols, cols);
}

// one thread per value: (value * s) / norm, rounded away from zero at ties
__global__ void __launch_bounds__(kThreads) scaled_value_kernel(const float *__restrict__ v, const float *__restrict__ norms,
                                                               long long rows, long long cols, float scale,
                                                               long long *__restrict__ out, int *bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    bool wrong = false;
    out[i] = procdb::pnns_scaled_value(v[i], scale, norms[i / cols], wrong);
    if (wrong) *bad = 1;
}

// Eval position j of query plaintext blockIdx.y takes SIMD slot inverse[j] of its .denseRow packing (encodeSimd's
// scatter as a gather); the signed value is mapped as PlaintextMatrix.init(signedValues:reduce:) maps it
__global__ void __launch_bounds__(kThreads) dense_row_kernel(const long long *__restrict__ values, long long rows,
                                                            long long cols, int logn, u64 t, int reduce,
                                                            const int32_t *__restrict__ inverse, u64 *__restrict__ out,
                                                            int *bad) {
    const int n = 1 << logn;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long p = blockIdx.y;
    const long long at = procdb::pnns_dense_row_element(rows, cols, logn, p, inverse[j]);
    u64 v = 0;
    if (at >= 0) {
        bool wrong = false;
        v = procdb::pnns_signed_value(values[at], t, reduce != 0, wrong);
        if (wrong) *bad = 1;
    }
    out[p * n + j] = v;
}

struct DistanceArgs {
    long long rows, cols, replies, scaling_factor;
    int logn;
    procdb::PnnsCrt crt;
};

// element (r, c) of the rows x cols distance matrix: its SIMD slot in every context's decoded replies (decoded:
// count x replies x N, context-major), the CRT composition, the centred value over prod t, the float epilogue
__global__ void __launch_bounds__(kThreads) distance_kernel(const u64 *__restrict__ decoded, const __grid_constant__ DistanceArgs a,
                                                           float *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.rows * a.cols) return;
    const long long r = i / a.cols, c = i - r * a.cols;
    long long p, slot;
    procdb::pnns_dense_column_slot(a.rows, a.cols, a.logn, r, c, p, slot);
    uint64_t x[kMaxPlaintextModuli];
    const long long per_context = a.replies << a.logn;
    for (int k = 0; k < a.crt.count; ++k) x[k] = decoded[k * per_context + (p << a.logn) + slot];
    out[i] = procdb::pnns_distance(procdb::pnns_crt_signed(a.crt, x), a.scaling_factor);
}

unsigned blocks(long long items) { return (unsigned)((items + kThreads - 1) / kThreads); }

// Device buffers of one call on one stream; the secret ones are zeroized before they are freed.
struct Buffers {
    cudaStream_t s;
    struct B {
        void *p;
        size_t bytes;
        bool secret;
    };
    std::vector<B> list;
    cudaError_t e = cudaSuccess;
    explicit Buffers(cudaStream_t st) : s(st) {}
    template <class T>
    T *get(size_t bytes, bool secret = false) {
        void *p = nullptr;
        if (e == cudaSuccess) e = cudaMallocAsync(&p, std::max<size_t>(bytes, 16), s);
        if (e != cudaSuccess) return nullptr;
        list.push_back({p, bytes, secret});
        return (T *)p;
    }
    ~Buffers() {
        for (const B &b : list) {
            if (b.secret) cudaMemsetAsync(b.p, 0, b.bytes, s);
            cudaFreeAsync(b.p, s);
        }
    }
};

int32_t finish(cudaStream_t s, cudaError_t e, const char *what) {
    const cudaError_t e2 = wait_stream(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, what);
}

}  // namespace

namespace hecuda {

cudaError_t launch_pnns_normalize(const float *vectors, int64_t rows, int64_t cols, int64_t scaling_factor, float *norms,
                                  int64_t *values, int *bad, cudaStream_t s) {
    if (rows == 0) return cudaSuccess;
    const cudaError_t e = launch(row_norm_kernel, blocks(rows), kThreads, 0, s, vectors, (long long)rows, (long long)cols, norms);
    if (e != cudaSuccess) return e;
    return launch(scaled_value_kernel, blocks(rows * cols), kThreads, 0, s, vectors, norms, (long long)rows, (long long)cols,
                  (float)scaling_factor, (long long *)values, bad);
}

namespace api {

int32_t check_float_vectors(const float *vectors, int64_t rows, int64_t cols, int64_t scaling_factor, u64 t, bool reduce,
                            bool scan) {
    if (!vectors) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (scaling_factor < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "scaling factor must not be negative");
    // |value * s / norm| <= s up to rounding: a scaling factor past the plaintext map's range cannot be honoured
    const double bound = reduce ? 4611686018427387904.0 : (double)((t - 1) / 2);
    if ((double)(float)scaling_factor > bound)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, reduce ? "scaling factor outside Int64" :
                                                          "scaling factor leaves [-floor(t/2), floor((t-1)/2)]");
    for (int64_t i = 0; scan && i < rows * cols; ++i)
        if (!std::isfinite(vectors[i])) return fail(HECUDA_ERR_INVALID_ARGUMENT, "non-finite vector value");
    return HECUDA_OK;
}

}  // namespace api
}  // namespace hecuda

extern "C" {

int32_t hecuda_pnns_query_generate(const hecuda_context *h, const uint64_t *secret_key, const float *vectors, int64_t row_count,
                                   int64_t column_count, int64_t scaling_factor, int32_t reduce, const uint8_t *a_seeds,
                                   const uint8_t *error_seeds, uint64_t *ciphertexts, uint8_t *poly0) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!secret_key) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (!a_seeds || !error_seeds || !ciphertexts == !poly0)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument: seeds and exactly one of ciphertexts / poly0");
    const Context &c = *h->ctx;
    if (!c.simd) return fail(HECUDA_ERR_UNSUPPORTED, "simdEncodingNotSupported");
    if (row_count < 1 || column_count < 1 || column_count > c.n / 2)  // PnnsError.invalidMatrixDimensions
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    if ((rc = check_float_vectors(vectors, row_count, column_count, scaling_factor, c.t, reduce != 0, true))) return rc;
    const int64_t count = procdb::pnns_dense_row_count(row_count, column_count, c.logn);
    if (count > kMaxGridYZ) return fail(HECUDA_ERR_INVALID_ARGUMENT, "too many query rows");  // grid y of dense_row_kernel
    const int L = c.L;
    const int64_t n = c.n;
    const size_t poly_words = (size_t)L * n, values = (size_t)row_count * column_count;
    CodecConsts cc;
    std::string err;
    if (poly0 && !codec_consts(c, c.map_q(L), 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const size_t poly_bytes = poly0 ? (size_t)serialized_poly_bytes(cc) : 0;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    cudaError_t e;
    int bad = 0;
    {
        Buffers m(s);
        float *d_vec = m.get<float>(values * sizeof(float), true);
        float *d_norm = m.get<float>((size_t)row_count * sizeof(float), true);
        int64_t *d_vals = m.get<int64_t>(values * sizeof(int64_t), true);
        int *d_bad = m.get<int>(sizeof(int));
        u64 *d_pt = m.get<u64>((size_t)count * n * sizeof(u64), true);
        u64 *d_sk = m.get<u64>(poly_words * sizeof(u64), true);
        unsigned char *d_as = m.get<unsigned char>((size_t)32 * count), *d_es = m.get<unsigned char>((size_t)32 * count, true);
        u64 *d_ct = m.get<u64>(2 * poly_words * count * sizeof(u64));
        unsigned char *d_bytes = poly0 ? m.get<unsigned char>(poly_bytes * count) : nullptr;
        e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_vec, vectors, values * sizeof(float), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0, sizeof(int), s);
        if (e == cudaSuccess) e = launch_pnns_normalize(d_vec, row_count, column_count, scaling_factor, d_norm, d_vals, d_bad, s);
        if (e == cudaSuccess)
            e = launch(dense_row_kernel, dim3(blocks(n), (unsigned)count), kThreads, 0, s, (const long long *)d_vals, row_count,
                       column_count, c.logn, c.t, reduce, c.d_simd_inverse, d_pt, d_bad);
        // encodeSimd's inverse NTT mod t (Encoding.swift:206-214)
        if (e == cudaSuccess) e = ntt_single(c, c.slot_t(), true, d_pt, d_pt, count, s);
        // a value Swift would trap on refuses the call before anything is encrypted or returned
        if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = wait_stream(s);
        if (e == cudaSuccess && !bad) {
            u64 *d_c0 = d_ct, *d_c1 = d_ct + poly_words * count;
            e = cudaMemcpyAsync(d_sk, secret_key, poly_words * sizeof(u64), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_as, a_seeds, (size_t)32 * count, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_es, error_seeds, (size_t)32 * count, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = encrypt_plaintexts_device(c, d_sk, d_pt, d_as, d_es, d_c0, d_c1, !poly0, count, s);
            if (e == cudaSuccess && poly0) {
                e = launch_poly_serialize(c, cc, 0, d_c0, d_bytes, count, s);
                if (e == cudaSuccess) e = cudaMemcpyAsync(poly0, d_bytes, poly_bytes * count, cudaMemcpyDeviceToHost, s);
            } else if (e == cudaSuccess) {
                const size_t pw = poly_words * sizeof(u64);
                e = cudaMemcpy2DAsync(ciphertexts, 2 * pw, d_c0, pw, pw, (size_t)count, cudaMemcpyDeviceToHost, s);
                if (e == cudaSuccess)
                    e = cudaMemcpy2DAsync(ciphertexts + poly_words, 2 * pw, d_c1, pw, pw, (size_t)count, cudaMemcpyDeviceToHost, s);
            }
        }
    }
    rc = finish(s, e, "pnns_query_generate");
    if (rc == HECUDA_OK && bad)  // Int64(_:) traps, or Scalar.centeredToRemainder's precondition (Scalar.swift:85-87)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "a scaled value leaves Int64 or the plaintext range; pass reduce to reduce mod t");
    return rc;
}

int32_t hecuda_pnns_decrypt_distances(const hecuda_context *const *ctxs, int32_t plaintext_count, const uint64_t *secret_key,
                                      const uint64_t *const *replies, int64_t reply_count, int32_t moduli_count,
                                      int64_t matrix_rows, int64_t query_rows, int64_t scaling_factor, float *distances) {
    if (!ctxs || plaintext_count < 1 || plaintext_count > kMaxPlaintextModuli)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "plaintext_count must be 1 .. 8 contexts");
    int32_t rc;
    for (int32_t k = 0; k < plaintext_count; ++k)
        if ((rc = check_ctx(ctxs[k]))) return rc;
    if (!secret_key) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (!replies || !distances) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    for (int32_t k = 0; k < plaintext_count; ++k)
        if (!replies[k]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *ctxs[0]->ctx;
    procdb::PnnsCrt crt{};
    crt.count = plaintext_count;
    unsigned __int128 product = 1;
    for (int32_t k = 0; k < plaintext_count; ++k) {
        const Context &ck = *ctxs[k]->ctx;
        bool same = ck.n == c.n && ck.L == c.L && ck.word_bits == c.word_bits;
        for (int i = 0; same && i < c.L; ++i) same = ck.q[i] == c.q[i];
        if (!same) return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongEncryptionParameters: the contexts differ in more than t");
        if (!ck.simd) return fail(HECUDA_ERR_UNSUPPORTED, "simdEncodingNotSupported");
        if (ck.t >= ck.gamma) return fail(HECUDA_ERR_UNSUPPORTED, "plaintext modulus too large");
        for (int32_t j = 0; j < k; ++j)
            if (crt.t[j] == ck.t) return fail(HECUDA_ERR_INVALID_ARGUMENT, "plaintext moduli must be pairwise distinct");
        crt.t[k] = ck.t;
        product *= ck.t;
    }
    // CrtComposer.compose's precondition: UInt64 holds composeMaxIntermediateValue = 2 prod t (CrtComposer.swift:54-79)
    if (plaintext_count > 1 && product > (unsigned __int128)(~0ull) / 2)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "2 * prod(plaintext moduli) exceeds UInt64.max");
    crt.product = (uint64_t)product;
    for (int32_t k = 0; k < plaintext_count; ++k) {
        crt.punct[k] = crt.product / crt.t[k];
        crt.inv[k] = host::invmod(crt.punct[k] % crt.t[k], crt.t[k]);
    }
    if (moduli_count < 1 || moduli_count > c.L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (matrix_rows < 1 || query_rows < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    const int64_t expected = procdb::pnns_dense_column_count(matrix_rows, query_rows, c.logn);
    if (reply_count != expected)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongCiphertextCount(got: " + std::to_string(reply_count) + ", expected: " +
                                                     std::to_string(expected) + ")");
    const int l = moduli_count;
    const int64_t n = c.n;
    const size_t in_words = (size_t)2 * l * n * reply_count, total = (size_t)matrix_rows * query_rows;
    WsGuard g(ctxs[0]);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    cudaError_t e;
    {
        Buffers m(s);
        u64 *d_sk = m.get<u64>((size_t)l * n * sizeof(u64), true);
        u64 *d_in = m.get<u64>(in_words * sizeof(u64));
        u64 *d_scratch = m.get<u64>(decrypt_scratch_words(c, 2, l) * reply_count * sizeof(u64), true);
        u64 *d_pt = m.get<u64>((size_t)reply_count * n * sizeof(u64), true);
        u64 *d_dec = m.get<u64>((size_t)plaintext_count * reply_count * n * sizeof(u64), true);
        float *d_out = m.get<float>(total * sizeof(float), true);
        e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_sk, secret_key, (size_t)l * n * sizeof(u64), cudaMemcpyHostToDevice, s);
        for (int32_t k = 0; e == cudaSuccess && k < plaintext_count; ++k) {
            const Context &ck = *ctxs[k]->ctx;
            // d_in is rewritten only after the previous context's decryption has read it (one stream)
            e = cudaMemcpyAsync(d_in, replies[k], in_words * sizeof(u64), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = decrypt_device(ck, d_sk, d_in, 2, l, d_scratch, d_pt, reply_count, s);
            if (e == cudaSuccess)
                e = launch_decode_simd(ck, d_pt, 0, d_dec + (size_t)k * reply_count * n, d_scratch, reply_count, s);
        }
        if (e == cudaSuccess) {
            const DistanceArgs a{matrix_rows, query_rows, reply_count, scaling_factor, c.logn, crt};
            e = launch(distance_kernel, blocks((long long)total), kThreads, 0, s, d_dec, a, d_out);
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(distances, d_out, total * sizeof(float), cudaMemcpyDeviceToHost, s);
    }
    return finish(s, e, "pnns_decrypt_distances");
}

}  // extern "C"
