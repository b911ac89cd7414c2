// client.cu -- the client side of BFV on the device: secret keys, symmetric encryption and evaluation keys.
//
//   Bfv.generateSecretKey              Bfv/Bfv+Keys.swift:20-26     (randomizeTernary, PolyRq+Randomize.swift:87-104)
//   Bfv.encrypt = encryptZero + Add    Bfv/Bfv+Encrypt.swift:64-72, 141-181 (plaintextTranslate :75-139)
//   Bfv.generateEvaluationKey          Bfv/Bfv+Keys.swift:30-65     (_generateKeySwitchKey :67-103)
//
// Every random polynomial comes from a NistAes128Ctr stream keyed by a 32-byte seed the caller supplies: the uniform `a`
// (as the reference), and also the secret and the error, which the reference draws from SystemRandomNumberGenerator.
// The chains of 4096-byte segments come from drbg.cu; the kernels here read a coefficient's bytes straight from its
// segment (sampling.cuh).  Encryption is three launches per chunk: `a` and a * s (Eval) from the a-stream in one kernel,
// one inverse NTT over both, then one epilogue that samples the error and applies -(. + e) + Delta m + adjust in
// registers.  The error never exists in HBM during encryption; key copies and the key-switching errors are zeroized
// before they are freed.
#include <algorithm>
#include <vector>

#include "capi_internal.hpp"
#include "sampling.cuh"

using namespace hecuda;
using namespace hecuda::api;
using namespace hecuda::drbg;

namespace {

constexpr int kThreads = 256;
constexpr double kErrorStdDev = 3.2;  // ErrorStdDev.stdDev32, the only value EncryptionParameters accepts as secure

struct RowConsts {
    int rows;
    u64 p[kMaxRows];
    u64 ks_mod[kMaxRows];  // q_ks mod p_r (_generateKeySwitchKey's modulusProduct, Bfv+Keys.swift:87-90)
};

struct Tables {
    const unsigned char *sbox;
    const u32w *te0;
};

__device__ __forceinline__ void load_tables(const Tables &g, unsigned char *sbox, u32w *te0) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        sbox[i] = g.sbox[i];
        te0[i] = g.te0[i];
    }
    __syncthreads();
}

__device__ __forceinline__ StreamReader reader(const u32w *rk, const u64 *ctr, int segments, long long seed,
                                               const unsigned char *sbox, const u32w *te0) {
    StreamReader st;
    st.rk = rk + (size_t)seed * segments * kRoundKeyWords;
    st.ctr = ctr + (size_t)seed * segments * 2;
    st.sbox = sbox;
    st.te0 = te0;
    return st;
}

__device__ __forceinline__ u64 mulmod(u64 a, u64 b, u64 p) { return (u64)(((u128)a * b) % p); }

// the uniform coefficient k of a stream: its k-th little-endian 128-bit word mod p (randomizeUniform, :56-75)
__device__ __forceinline__ u64 uniform_value(StreamReader &st, long long k, u64 p) {
    const u64 lo = st.word64(16 * k), hi = st.word64(16 * k + 8);
    return (u64)((((u128)hi << 64) | lo) % p);
}

// secret keys: coefficient j of seed blockIdx.y, val - 1 on every row (randomizeTernary), Coeff format
__global__ void __launch_bounds__(kThreads) ternary_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr, int segments,
                                                           const __grid_constant__ Tables g, const __grid_constant__ RowConsts c,
                                                           u64 *__restrict__ out, int n) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    StreamReader st = reader(rk, ctr, segments, blockIdx.y, sbox, te0);
    const long long v = (long long)ternary_value(st, j) - 1;
    u64 *dst = out + (size_t)blockIdx.y * c.rows * n + j;
    for (int r = 0; r < c.rows; ++r) dst[(size_t)r * n] = signed_residue(v, c.p[r]);
}

// errors of key-switching ciphertexts: coefficient j of seed blockIdx.y on every row (randomizeCenteredBinomial...)
__global__ void __launch_bounds__(kThreads) cbd_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr, int segments,
                                                       const __grid_constant__ Tables g, const __grid_constant__ RowConsts c,
                                                       int words, u64 mask, u64 *__restrict__ out, int n) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    StreamReader st = reader(rk, ctr, segments, blockIdx.y, sbox, te0);
    const int v = cbd_value(st, j, words, mask);
    u64 *dst = out + (size_t)blockIdx.y * c.rows * n + j;
    for (int r = 0; r < c.rows; ++r) dst[(size_t)r * n] = signed_residue(v, c.p[r]);
}

// encryptZero's Eval half for ciphertext blockIdx.y: a from its a-stream, a_s = a * s (PolyRq.mulAssign(secretPoly:))
__global__ void __launch_bounds__(kThreads) uniform_times_secret_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr,
                                                                        int segments, const __grid_constant__ Tables g,
                                                                        const __grid_constant__ RowConsts c,
                                                                        const u64 *__restrict__ sk, u64 *__restrict__ a_s,
                                                                        u64 *__restrict__ a, int n) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)c.rows * n) return;
    StreamReader st = reader(rk, ctr, segments, blockIdx.y, sbox, te0);
    const u64 p = c.p[k / n];
    const u64 v = uniform_value(st, k, p);
    const size_t o = (size_t)blockIdx.y * c.rows * n + k;
    a[o] = v;
    a_s[o] = mulmod(v, sk[k], p);
}

// the encryption epilogue, after the inverse NTT of a * s: c0 = -(c0 + e) + (Delta m + adjust) with e sampled from
// ciphertext blockIdx.y's error stream (plaintextTranslate(.Add) with the translate constants of plaintext.cu)
__global__ void __launch_bounds__(kThreads) encrypt_epilogue_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr,
                                                                    int segments, const __grid_constant__ Tables g,
                                                                    const __grid_constant__ TranslateConsts tc, int words,
                                                                    u64 mask, const u64 *__restrict__ pt, u64 *__restrict__ c0,
                                                                    int n) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    StreamReader st = reader(rk, ctr, segments, blockIdx.y, sbox, te0);
    const int e = cbd_value(st, j, words, mask);
    const u64 m = pt[(size_t)blockIdx.y * n + j];
    const u64 adj = translate_adjust(m, tc);
    u64 *x = c0 + (size_t)blockIdx.y * tc.l * n + j;
    for (int r = 0; r < tc.l; ++r) {
        const u64 q = tc.q[r];
        const u64 noisy = add_mod(x[(size_t)r * n], signed_residue(e, q), q);
        x[(size_t)r * n] = sub_mod(add_mod(shoup_mul(m, tc.delta[r], tc.delta_p[r], q), adj, q), noisy, q);
    }
}

// _generateKeySwitchKey for key ciphertext ct = first + blockIdx.y (row i = ct mod L of key ct / L) over the K rows
// of the key-switching context, in Eval: poly1 = a, poly0 = -(a * s + NTT(e)) + [r == i] (q_ks mod q_r) cur[r].  poly0
// goes to the key and over its error (`e_poly0`, then a contiguous copy for serialization).
__global__ void __launch_bounds__(kThreads) key_switch_key_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr,
                                                                  int segments, const __grid_constant__ Tables g,
                                                                  const __grid_constant__ RowConsts c, int L,
                                                                  const u64 *__restrict__ sk, const u64 *__restrict__ cur,
                                                                  u64 *__restrict__ e_poly0, u64 *const *__restrict__ dst, int n,
                                                                  long long first) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long words = (long long)c.rows * n;
    if (k >= words) return;
    const long long ct = first + blockIdx.y;
    StreamReader st = reader(rk, ctr, segments, ct, sbox, te0);
    const int row = (int)(k / n), i = (int)(ct % L);
    const u64 p = c.p[row];
    const u64 a = uniform_value(st, k, p);
    const size_t o = (size_t)ct * words + k;
    u64 v = p - add_mod(mulmod(a, sk[k], p), e_poly0[o], p);
    v = v == p ? 0 : v;
    if (row == i) v = add_mod(v, mulmod(c.ks_mod[row], cur[(size_t)(ct / L) * words + k], p), p);
    e_poly0[o] = v;
    u64 *out = dst[ct];
    out[k] = v;
    out[words + k] = a;
}

__global__ void __launch_bounds__(kThreads) square_kernel(const u64 *__restrict__ s, u64 *__restrict__ out,
                                                          const __grid_constant__ RowConsts c, int n) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)c.rows * n) return;
    out[k] = mulmod(s[k], s[k], c.p[k / n]);
}

// ---------------------------------------------------------------- host side

RowConsts row_consts(const Context &c, const NttRowMap &map, int rows) {
    RowConsts rc{};
    rc.rows = rows;
    for (int r = 0; r < rows; ++r) {
        rc.p[r] = c.slots[map.slot[r]].dev.p;
        rc.ks_mod[r] = c.has_ks ? c.q_ks % rc.p[r] : 0;
    }
    return rc;
}

int segments_for(long long bytes) { return (int)((bytes + kSegmentBytes - 1) / kSegmentBytes); }

// The chains of `count` seeds already on the device; the round keys are zeroized when it goes out of scope.
struct Streams {
    u32w *rk = nullptr;
    u64 *ctr = nullptr;
    int segments = 0;
    int64_t count = 0;
    cudaStream_t s = nullptr;
    cudaError_t make(const unsigned char *d_seeds, int segs, int64_t n, cudaStream_t st) {
        segments = segs, count = n, s = st;
        return drbg_chains(d_seeds, segs, n, &rk, &ctr, st);
    }
    ~Streams() {
        if (s) free_chains(rk, ctr, segments, count, s);
    }
};

// Device buffers of one call, on one stream; the ones marked secret are zeroized before they are freed.
struct Allocs {
    cudaStream_t s;
    struct A {
        void *p;
        size_t bytes;
        bool secret;
    };
    std::vector<A> list;
    cudaError_t e = cudaSuccess;
    explicit Allocs(cudaStream_t st) : s(st) {}
    template <class T>
    T *get(size_t bytes, bool secret = false) {
        void *p = nullptr;
        if (e == cudaSuccess) e = cudaMallocAsync(&p, std::max<size_t>(bytes, 16), s);
        if (e != cudaSuccess) return nullptr;
        list.push_back({p, bytes, secret});
        return (T *)p;
    }
    ~Allocs() {
        for (const A &a : list) {
            if (a.secret) cudaMemsetAsync(a.p, 0, a.bytes, s);
            cudaFreeAsync(a.p, s);
        }
    }
};

int32_t finish(cudaStream_t s, cudaError_t e, const char *what) {
    const cudaError_t e2 = wait_stream(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, what);
}

int secret_rows(const Context &c) { return c.has_ks ? c.L + 1 : c.L; }
NttRowMap secret_map(const Context &c) { return c.has_ks ? c.map_ks(c.L) : c.map_q(c.L); }

cudaError_t tables(Tables &t) { return drbg_tables(&t.sbox, &t.te0); }

// Bfv.encrypt of `batch` plaintexts at the top level into d_c0 (batch x L x N) and, unless c1 is skipped, d_c1: the a
// and a * s kernel, the inverse NTT, the error + translate epilogue
cudaError_t encrypt_device(const Context &c, const u64 *d_sk, const u64 *d_pt, const unsigned char *d_a_seeds,
                           const unsigned char *d_e_seeds, u64 *d_c0, u64 *d_c1, bool c1_coeff, int64_t batch, cudaStream_t s) {
    const int L = c.L, n = (int)c.n;
    const NttRowMap map = c.map_q(L);
    const RowConsts rc = row_consts(c, map, L);
    int words = 0;
    u64 mask = 0;
    cbd_shape(kErrorStdDev, words, mask);
    Tables tb;
    cudaError_t e = tables(tb);
    Streams as, es;
    if (e == cudaSuccess) e = as.make(d_a_seeds, segments_for(16LL * L * n), batch, s);
    if (e == cudaSuccess) e = es.make(d_e_seeds, segments_for(8LL * words * n), batch, s);
    const unsigned gx = (unsigned)((L * (long long)n + kThreads - 1) / kThreads), gn = (unsigned)((n + kThreads - 1) / kThreads);
    if (e == cudaSuccess)
        e = for_each_part(batch, [&](int64_t first, int64_t part) {
            return launch(uniform_times_secret_kernel, dim3(gx, (unsigned)part), kThreads, 0, s,
                          as.rk + (size_t)first * as.segments * kRoundKeyWords, as.ctr + (size_t)first * as.segments * 2,
                          as.segments, tb, rc, d_sk, d_c0 + (size_t)first * L * n, d_c1 + (size_t)first * L * n, n);
        });
    // c0 and c1 are adjacent: one inverse NTT over both (c0 alone when only poly0 is wanted)
    if (e == cudaSuccess) e = launch_ntt_inverse(c, map, d_c0, d_c0, batch * L * (c1_coeff ? 2 : 1), kScalePlain, s);
    if (e == cudaSuccess)
        e = for_each_part(batch, [&](int64_t first, int64_t part) {
            return launch(encrypt_epilogue_kernel, dim3(gn, (unsigned)part), kThreads, 0, s,
                          es.rk + (size_t)first * es.segments * kRoundKeyWords, es.ctr + (size_t)first * es.segments * 2,
                          es.segments, tb, c.translate[L], words, mask, d_pt + (size_t)first * n, d_c0 + (size_t)first * L * n, n);
        });
    return e;
}

int32_t check_encrypt(const hecuda_context *h, const uint64_t *sk, const uint64_t *pt, const uint8_t *a_seeds,
                      const uint8_t *e_seeds, const void *out, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!sk) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (batch < 0 || (batch && (!pt || !a_seeds || !e_seeds || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    const Context &c = *h->ctx;
    for (int64_t i = 0; i < batch * c.n; ++i)
        if (pt[i] >= c.t) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPlaintext: coefficient >= plaintext modulus");
    return HECUDA_OK;
}

// Bfv.encrypt with host buffers; exactly one of ciphertexts (batch x 2 x L x N) / poly0 (batch x B bytes) is non-null
int32_t encrypt(const hecuda_context *h, const uint64_t *sk, const uint64_t *pt, const uint8_t *a_seeds, const uint8_t *e_seeds,
                uint64_t *ciphertexts, uint8_t *poly0, int64_t batch) {
    const Context &c = *h->ctx;
    const int L = c.L;
    const size_t poly_words = (size_t)L * c.n;
    CodecConsts cc;
    std::string err;
    if (poly0 && !codec_consts(c, c.map_q(L), 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const size_t poly_bytes = poly0 ? (size_t)serialized_poly_bytes(cc) : 0;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    const int64_t chunk = std::min<int64_t>(batch, std::max<int64_t>(1, (int64_t)((size_t)32 * 1024 * 1024 / (2 * poly_words))));
    cudaError_t e;
    {
        Allocs m(s);
        u64 *d_sk = m.get<u64>(poly_words * sizeof(u64), true);
        u64 *d_pt = m.get<u64>((size_t)chunk * c.n * sizeof(u64));
        unsigned char *d_as = m.get<unsigned char>((size_t)32 * chunk), *d_es = m.get<unsigned char>((size_t)32 * chunk, true);
        u64 *d_ct = m.get<u64>(2 * poly_words * chunk * sizeof(u64));
        unsigned char *d_bytes = poly0 ? m.get<unsigned char>(poly_bytes * chunk) : nullptr;
        e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_sk, sk, poly_words * sizeof(u64), cudaMemcpyHostToDevice, s);
        for (int64_t done = 0; e == cudaSuccess && done < batch; done += chunk) {
            const int64_t items = std::min<int64_t>(chunk, batch - done);
            u64 *d_c0 = d_ct, *d_c1 = d_ct + poly_words * items;
            e = cudaMemcpyAsync(d_pt, pt + (size_t)c.n * done, (size_t)c.n * items * sizeof(u64), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_as, a_seeds + 32 * done, (size_t)32 * items, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_es, e_seeds + 32 * done, (size_t)32 * items, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = encrypt_device(c, d_sk, d_pt, d_as, d_es, d_c0, d_c1, !poly0, items, s);
            if (e == cudaSuccess && poly0) {
                e = launch_poly_serialize(c, cc, 0, d_c0, d_bytes, items, s);
                if (e == cudaSuccess)
                    e = cudaMemcpyAsync(poly0 + poly_bytes * done, d_bytes, poly_bytes * items, cudaMemcpyDeviceToHost, s);
            } else if (e == cudaSuccess) {
                const size_t pw = poly_words * sizeof(u64);
                uint64_t *dst = ciphertexts + 2 * poly_words * done;
                e = cudaMemcpy2DAsync(dst, 2 * pw, d_c0, pw, pw, (size_t)items, cudaMemcpyDeviceToHost, s);
                if (e == cudaSuccess) e = cudaMemcpy2DAsync(dst + poly_words, 2 * pw, d_c1, pw, pw, (size_t)items, cudaMemcpyDeviceToHost, s);
            }
            // the next chunk's uploads overwrite d_pt / the seeds only after this chunk's kernels (one stream)
        }
    }
    return finish(s, e, poly0 ? "encrypt_seeded" : "encrypt");
}

}  // namespace

namespace hecuda {
namespace api {

cudaError_t encrypt_plaintexts_device(const Context &c, const u64 *d_sk, const u64 *d_pt, const unsigned char *d_a_seeds,
                                      const unsigned char *d_e_seeds, u64 *d_c0, u64 *d_c1, bool c1_coeff, int64_t batch,
                                      cudaStream_t s) {
    return encrypt_device(c, d_sk, d_pt, d_a_seeds, d_e_seeds, d_c0, d_c1, c1_coeff, batch, s);
}

}  // namespace api
}  // namespace hecuda

extern "C" {

int32_t hecuda_bfv_generate_secret_key(const hecuda_context *h, const uint8_t *seeds, uint64_t *secret_keys, int64_t count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (count < 0 || (count && (!seeds || !secret_keys))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    if (count == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const int rows = secret_rows(c), n = (int)c.n;
    const NttRowMap map = secret_map(c);
    const RowConsts rcs = row_consts(c, map, rows);
    const size_t words = (size_t)rows * n * count;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    cudaError_t e;
    {
        Allocs m(s);
        unsigned char *d_seeds = m.get<unsigned char>((size_t)32 * count, true);
        u64 *d_sk = m.get<u64>(words * sizeof(u64), true);
        e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_seeds, seeds, (size_t)32 * count, cudaMemcpyHostToDevice, s);
        Tables tb;
        if (e == cudaSuccess) e = tables(tb);
        Streams st;
        if (e == cudaSuccess) e = st.make(d_seeds, segments_for((long long)kTernaryBytes * n), count, s);
        if (e == cudaSuccess)
            e = for_each_part(count, [&](int64_t first, int64_t part) {
                return launch(ternary_kernel, dim3((unsigned)((n + kThreads - 1) / kThreads), (unsigned)part), kThreads, 0, s,
                              st.rk + (size_t)first * st.segments * kRoundKeyWords, st.ctr + (size_t)first * st.segments * 2,
                              st.segments, tb, rcs, d_sk + (size_t)first * rows * n, n);
            });
        if (e == cudaSuccess) e = launch_ntt_forward(c, map, d_sk, d_sk, count * rows, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(secret_keys, d_sk, words * sizeof(u64), cudaMemcpyDeviceToHost, s);
    }
    return finish(s, e, "generate_secret_key");
}

int32_t hecuda_bfv_encrypt(const hecuda_context *h, const uint64_t *secret_key, const uint64_t *plaintexts, const uint8_t *a_seeds,
                           const uint8_t *error_seeds, uint64_t *ciphertexts, int64_t batch) {
    int32_t rc = check_encrypt(h, secret_key, plaintexts, a_seeds, error_seeds, ciphertexts, batch);
    if (rc || batch == 0) return rc;
    return encrypt(h, secret_key, plaintexts, a_seeds, error_seeds, ciphertexts, nullptr, batch);
}

int32_t hecuda_bfv_encrypt_seeded(const hecuda_context *h, const uint64_t *secret_key, const uint64_t *plaintexts,
                                  const uint8_t *a_seeds, const uint8_t *error_seeds, uint8_t *poly0, int64_t batch) {
    int32_t rc = check_encrypt(h, secret_key, plaintexts, a_seeds, error_seeds, poly0, batch);
    if (rc || batch == 0) return rc;
    return encrypt(h, secret_key, plaintexts, a_seeds, error_seeds, nullptr, poly0, batch);
}

int32_t hecuda_evk_generate(const hecuda_context *h, const uint64_t *secret_key, int32_t has_relin, const uint32_t *elements,
                            int32_t element_count, const uint8_t *a_seeds, const uint8_t *error_seeds, hecuda_evk **out,
                            uint8_t *wire_poly0) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    const Context &c = *h->ctx;
    if (!c.has_ks)
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: a single coefficient modulus leaves no key-switching modulus");
    if (!secret_key) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (element_count < 0 || (element_count > 0 && !elements)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const int64_t keys = (has_relin ? 1 : 0) + element_count, count = keys * c.L;  // key ciphertexts
    if (count > 0 && (!a_seeds || !error_seeds)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null seeds");
    std::vector<uint32_t> sorted(elements, elements + element_count);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t el : sorted)
        if (!((el & 1) && el > 1 && el < 2 * c.n))  // isValidGaloisElement, Galois.swift:100-105
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid Galois element " + std::to_string(el));
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "repeated Galois element " + std::to_string(*std::adjacent_find(sorted.begin(), sorted.end())));
    const int K = c.L + 1, n = (int)c.n;
    const NttRowMap map = c.map_ks(c.L);
    const RowConsts rcs = row_consts(c, map, K);
    CodecConsts cc;
    std::string err;
    if (wire_poly0 && !codec_consts(c, map, 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    hecuda_evk *k = nullptr;
    if ((rc = hecuda_evk_create_empty(h, &k))) return rc;
    // key ciphertext i of key j lands at key_j + i x 2 x K x N: the relinearization key, then galois[elements[j]]
    std::vector<u64 *> dst;
    const size_t key_words = (size_t)K * n, ct_words = 2 * key_words;
    cudaError_t e = cudaSuccess;
    for (int32_t j = has_relin ? -1 : 0; j < element_count && e == cudaSuccess; ++j) {
        u64 *key = k->d_relin;
        if (j >= 0 && (e = cudaMalloc(&key, k->words * sizeof(u64))) == cudaSuccess) k->galois[elements[j]] = key;
        for (int i = 0; e == cudaSuccess && i < c.L; ++i) dst.push_back(key + ct_words * i);
    }
    if (e == cudaSuccess && count > 0) {
        WsGuard g(h);
        if (!g.w) {
            hecuda_evk_destroy(k);
            return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
        }
        cudaStream_t s = g.w->stream;
        {
            Allocs m(s);
            u64 *d_sk = m.get<u64>(key_words * sizeof(u64), true);
            u64 *d_cur = m.get<u64>(key_words * keys * sizeof(u64), true);  // s^2, then s(X^g) per element
            u64 *d_e = m.get<u64>(key_words * count * sizeof(u64), true);   // NTT(e), then poly0
            unsigned char *d_as = m.get<unsigned char>((size_t)32 * count), *d_es = m.get<unsigned char>((size_t)32 * count, true);
            u64 **d_dst = m.get<u64 *>(sizeof(u64 *) * count);
            unsigned char *d_bytes = wire_poly0 ? m.get<unsigned char>((size_t)serialized_poly_bytes(cc) * count) : nullptr;
            e = m.e;
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_sk, secret_key, key_words * sizeof(u64), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_as, a_seeds, (size_t)32 * count, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_es, error_seeds, (size_t)32 * count, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_dst, dst.data(), sizeof(u64 *) * count, cudaMemcpyHostToDevice, s);
            // currentKey of every key: s * s (generateRelinearizationKey, :58-65), s.applyGalois(element:) (:40-44)
            u64 *cur = d_cur;
            if (e == cudaSuccess && has_relin) {
                e = launch(square_kernel, (unsigned)((key_words + kThreads - 1) / kThreads), kThreads, 0, s, d_sk, cur, rcs, n);
                cur += key_words;
            }
            for (int32_t j = 0; e == cudaSuccess && j < element_count; ++j, cur += key_words)
                e = launch_galois_eval(c, K, elements[j], d_sk, cur, 1, s);
            int words = 0;
            u64 mask = 0;
            cbd_shape(kErrorStdDev, words, mask);
            Tables tb;
            if (e == cudaSuccess) e = tables(tb);
            {
                Streams es;
                if (e == cudaSuccess) e = es.make(d_es, segments_for(8LL * words * n), count, s);
                if (e == cudaSuccess)
                    e = for_each_part(count, [&](int64_t first, int64_t part) {
                        return launch(cbd_kernel, dim3((unsigned)((n + kThreads - 1) / kThreads), (unsigned)part), kThreads, 0, s,
                                      es.rk + (size_t)first * es.segments * kRoundKeyWords,
                                      es.ctr + (size_t)first * es.segments * 2, es.segments, tb, rcs, words, mask,
                                      d_e + key_words * first, n);
                    });
            }
            if (e == cudaSuccess) e = launch_ntt_forward(c, map, d_e, d_e, count * K, s);
            Streams as;
            if (e == cudaSuccess) e = as.make(d_as, segments_for(16LL * K * n), count, s);
            if (e == cudaSuccess)
                e = for_each_part(count, [&](int64_t first, int64_t part) {
                    return launch(key_switch_key_kernel, dim3((unsigned)((key_words + kThreads - 1) / kThreads), (unsigned)part),
                                  kThreads, 0, s, as.rk, as.ctr, as.segments, tb, rcs, c.L, d_sk, d_cur, d_e, d_dst, n, first);
                });
            if (e == cudaSuccess && wire_poly0) {
                const size_t b = (size_t)serialized_poly_bytes(cc);
                e = launch_poly_serialize(c, cc, 0, d_e, d_bytes, count, s);
                if (e == cudaSuccess) e = cudaMemcpyAsync(wire_poly0, d_bytes, b * count, cudaMemcpyDeviceToHost, s);
            }
        }
        // the keys are read on other non-blocking streams: return once the kernels have written them (see upload())
        const cudaError_t e2 = wait_stream(s);
        if (e == cudaSuccess) e = e2;
    }
    if (e != cudaSuccess) {
        hecuda_evk_destroy(k);
        return cuda_fail(e, "evk_generate");
    }
    k->loaded = has_relin != 0;
    *out = k;
    return HECUDA_OK;
}

}  // extern "C"
