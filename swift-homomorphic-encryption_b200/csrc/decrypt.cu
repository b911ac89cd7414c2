// decrypt.cu -- BFV decryption on the device (SURVEY.md 8f rank 4).
//
//   Bfv.decryptCoeff / decryptEval     Bfv/Bfv+Decrypt.swift:21-41   (dotProduct(ciphertext:with:) :188-204)
//   RnsTool.scaleAndRound              RnsTool.swift:272-302         (BEHZ Algorithm 2, eprint 2016/510)
//
// c_0 + c_1 s + c_2 s^2 in Eval format, inverse NTT, then per coefficient: scale by gamma*t, exact base conversion to
// {t, gamma} (the sums are reduced modulo the small moduli, so any summation order gives the reference's residues),
// the gamma-centred correction, and the final multiplication by gamma^-1 * scalingFactor mod t.
#include <cmath>
#include <vector>

#include "capi_internal.hpp"
#include "hostmath.hpp"
#include "modarith.cuh"

using namespace hecuda;
using namespace hecuda::api;

namespace {

// gamma = T.rnsCorrectionFactor comes from the context: 2^62 - 40797 (UInt64) or 2^30 - 20405 (UInt32), Scalar.swift:503-520

struct DecryptConsts {
    int l;
    u64 t;
    u64 gamma;                 // T.rnsCorrectionFactor
    u64 q[kMaxL];
    u64 gamma_t[kMaxL];        // gamma * t mod q_i                       (prodGammaTModQ, RnsTool.swift:145-146)
    u64 inv_punctured[kMaxL];  // (q / q_i)^-1 mod q_i                    (RnsBaseConverter)
    u64 punctured_t[kMaxL];    // q / q_i mod t
    u64 punctured_g[kMaxL];    // q / q_i mod gamma
    u64 neg_inv_q_t, neg_inv_q_g;  // -q^-1 mod t, mod gamma             (negInverseQModTGamma, :154-157)
    u64 inv_gamma_scaled;      // gamma^-1 * scalingFactor mod t          (:147-150, :298-299)
};

__device__ __forceinline__ u64 mulmod_dev(u64 a, u64 b, u64 m) { return (u64)(((u128)a * b) % m); }

// d = c_0 + sum_k c_k s^k (Eval), one thread per (item, row, coefficient)
__global__ void __launch_bounds__(256) dot_secret_kernel(const u64 *__restrict__ ct, const u64 *__restrict__ sk,
                                                        u64 *__restrict__ out, const __grid_constant__ DecryptConsts c,
                                                        int n, int polys) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int row = blockIdx.y;
    const int64_t item = blockIdx.z;
    const u64 q = c.q[row];
    const u64 s = sk[(int64_t)row * n + e];
    const u64 *src = ct + (item * polys * c.l + row) * (int64_t)n + e;
    u64 acc = src[0], power = s;
    for (int k = 1; k < polys; ++k) {
        const u64 term = mulmod_dev(src[(int64_t)k * c.l * n], power, q);
        acc = acc + term >= q ? acc + term - q : acc + term;
        power = mulmod_dev(power, s, q);
    }
    out[(item * c.l + row) * (int64_t)n + e] = acc;
}

__global__ void __launch_bounds__(256) scale_and_round_kernel(const u64 *__restrict__ dot, u64 *__restrict__ out,
                                                             const __grid_constant__ DecryptConsts c, int n) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int64_t item = blockIdx.y;
    u64 mod_t = 0, mod_g = 0;
    for (int i = 0; i < c.l; ++i) {
        const u64 x = mulmod_dev(dot[(item * c.l + i) * (int64_t)n + e], c.gamma_t[i], c.q[i]);
        const u64 y = mulmod_dev(x, c.inv_punctured[i], c.q[i]);
        mod_t = (mod_t + mulmod_dev(y % c.t, c.punctured_t[i], c.t)) % c.t;
        mod_g = (u64)(((u128)mod_g + mulmod_dev(y % c.gamma, c.punctured_g[i], c.gamma)) % c.gamma);
    }
    mod_t = mulmod_dev(mod_t, c.neg_inv_q_t, c.t);
    mod_g = mulmod_dev(mod_g, c.neg_inv_q_g, c.gamma);
    const u64 s_greater = (c.t - (c.gamma - mod_g) % c.t) % c.t;
    const u64 s_less = mod_g % c.t;
    const u64 s = mod_g > c.gamma / 2 ? s_greater : s_less;
    const u64 m = mod_t >= s ? mod_t - s : mod_t + c.t - s;
    out[item * (int64_t)n + e] = mulmod_dev(m, c.inv_gamma_scaled, c.t);
}

DecryptConsts make_consts(const Context &ctx, int l, u64 scaling_factor) {
    DecryptConsts c;
    c.l = l;
    c.t = ctx.t;
    const u64 kGamma = c.gamma = ctx.gamma;
    u64 q[kMaxL];
    for (int i = 0; i < l; ++i) q[i] = c.q[i] = ctx.slots[ctx.slot_q(i)].dev.p;
    for (int i = 0; i < l; ++i) {
        c.gamma_t[i] = host::mulmod(kGamma % q[i], ctx.t % q[i], q[i]);
        c.inv_punctured[i] = host::invmod(host::punctured_mod(q, l, i, q[i]), q[i]);
        c.punctured_t[i] = host::punctured_mod(q, l, i, ctx.t);
        c.punctured_g[i] = host::punctured_mod(q, l, i, kGamma);
    }
    const u64 q_t = host::prod_mod(q, l, ctx.t), q_g = host::prod_mod(q, l, kGamma);
    c.neg_inv_q_t = (ctx.t - host::invmod(q_t, ctx.t)) % ctx.t;
    c.neg_inv_q_g = (kGamma - host::invmod(q_g, kGamma)) % kGamma;
    c.inv_gamma_scaled = host::mulmod(host::invmod(kGamma % ctx.t, ctx.t), scaling_factor % ctx.t, ctx.t);
    return c;
}

cudaError_t decrypt_chunk(const Context &c, const DecryptConsts &dc, u64 *scratch, const u64 *sk, const u64 *ct, int polys,
                          u64 *out, int64_t items, cudaStream_t s) {
    const int l = dc.l;
    const int64_t n = c.n;
    u64 *ev = scratch, *dot = scratch + (size_t)items * polys * l * n;
    const NttRowMap map = c.map_q(l);
    cudaError_t e;
    if ((e = launch_ntt_forward(c, map, ct, ev, items * polys * l, s)) != cudaSuccess) return e;
    const int threads = coeff_threads(n);
    const unsigned gx = (unsigned)((n + threads - 1) / threads);
    e = for_each_part(items, [&](int64_t done, int64_t part) {
        return launch(dot_secret_kernel, dim3(gx, (unsigned)l, (unsigned)part), threads, 0, s, ev + done * polys * l * n, sk,
                      dot + done * l * n, dc, (int)n, polys);
    });
    if (e != cudaSuccess) return e;
    if ((e = launch_ntt_inverse(c, map, dot, dot, items * l, kScalePlain, s)) != cudaSuccess) return e;
    return for_each_part(items, [&](int64_t done, int64_t part) {
        return launch(scale_and_round_kernel, dim3(gx, (unsigned)part), threads, 0, s, dot + done * l * n, out + done * n, dc,
                      (int)n);
    });
}

// ---------------------------------------------------------------- noise budget
// Bfv.noiseBudgetEval (Bfv+Decrypt.swift:116-174): v = c_0 + c_1 s (+ c_2 s^2) by dot_secret_kernel, the inverse NTT,
// then per coefficient the CRT composition of [v t]_{q_i} into a multi-word integer in [0, q) (RnsTool.crtCompose),
// its centred absolute value against (q + 1) / 2, and the maximum over the ciphertext.  The host turns the maximum into
// log2(qDouble / (2 norm)).
constexpr int kNormThreads = 256;

struct NoiseConsts {
    int l;              // rows = words of q (every q_i < 2^64)
    u64 q[kMaxL];
    u64 t_mod[kMaxL];   // t mod q_i
    u64 inv_punctured[kMaxL];  // (q / q_i)^-1 mod q_i
};

// a > b over `w` words (little-endian)
__device__ __forceinline__ bool wide_greater(const u64 *a, const u64 *b, int w) {
    for (int i = w - 1; i >= 0; --i)
        if (a[i] != b[i]) return a[i] > b[i];
    return false;
}

// one CTA per ciphertext; big = [q / q_i for each i][q][(q + 1) / 2], l words each; out: items x l words
__global__ void __launch_bounds__(kNormThreads) noise_norm_kernel(const u64 *__restrict__ v, const u64 *__restrict__ big,
                                                                 const __grid_constant__ NoiseConsts c, int n, u64 *__restrict__ out) {
    __shared__ u64 warp_best[kNormThreads / 32][kMaxL];
    const int W = c.l;
    const u64 *q = big + (size_t)W * W, *half = q + W;
    const long long item = blockIdx.x;
    u64 best[kMaxL], acc[kMaxL + 1], other[kMaxL];
    for (int w = 0; w < W; ++w) best[w] = 0;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        for (int w = 0; w <= W; ++w) acc[w] = 0;
        for (int i = 0; i < W; ++i) {
            const u64 x = v[(item * W + i) * (long long)n + e];
            const u64 y = mulmod_dev(mulmod_dev(x, c.t_mod[i], c.q[i]), c.inv_punctured[i], c.q[i]);
            const u64 *punct = big + (size_t)i * W;
            u64 carry = 0;
            for (int w = 0; w < W; ++w) {
                const u128 prod = (u128)y * punct[w] + acc[w] + carry;
                acc[w] = (u64)prod;
                carry = (u64)(prod >> 64);
            }
            acc[W] += carry;
        }
        // the sum is below l q: subtract q until it is in [0, q)
        while (acc[W] || !wide_greater(q, acc, W)) {
            u64 borrow = 0;
            for (int w = 0; w < W; ++w) {
                const u64 d = acc[w] - q[w] - borrow;
                borrow = (acc[w] < q[w] || (acc[w] == q[w] && borrow)) ? 1 : 0;
                acc[w] = d;
            }
            acc[W] -= borrow;
        }
        if (wide_greater(acc, half, W)) {  // q - coeff
            u64 borrow = 0;
            for (int w = 0; w < W; ++w) {
                const u64 d = q[w] - acc[w] - borrow;
                borrow = (q[w] < acc[w] || (q[w] == acc[w] && borrow)) ? 1 : 0;
                acc[w] = d;
            }
        }
        if (wide_greater(acc, best, W))
            for (int w = 0; w < W; ++w) best[w] = acc[w];
    }
    for (int off = 16; off > 0; off >>= 1) {
        for (int w = 0; w < W; ++w) other[w] = __shfl_down_sync(0xffffffffu, best[w], off);
        if (wide_greater(other, best, W))
            for (int w = 0; w < W; ++w) best[w] = other[w];
    }
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0)
        for (int w = 0; w < W; ++w) warp_best[warp][w] = best[w];
    __syncthreads();
    if (threadIdx.x) return;
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
        if (wide_greater(warp_best[k], best, W))
            for (int w = 0; w < W; ++w) best[w] = warp_best[k][w];
    for (int w = 0; w < W; ++w) out[item * W + w] = best[w];
}

// big = [q / q_i for each i][q][(q + 1) / 2] as l-word integers
std::vector<u64> noise_big_constants(const u64 *q, int l) {
    std::vector<u64> big((size_t)(l + 2) * l, 0);
    auto mul_small = [&](u64 *x, u64 m) {
        u64 carry = 0;
        for (int w = 0; w < l; ++w) {
            const unsigned __int128 p = (unsigned __int128)x[w] * m + carry;
            x[w] = (u64)p;
            carry = (u64)(p >> 64);
        }
    };
    for (int i = 0; i < l; ++i) {
        u64 *p = &big[(size_t)i * l];
        p[0] = 1;
        for (int j = 0; j < l; ++j)
            if (j != i) mul_small(p, q[j]);
    }
    u64 *prod = &big[(size_t)l * l], *half = prod + l;
    prod[0] = 1;
    for (int j = 0; j < l; ++j) mul_small(prod, q[j]);
    unsigned carry = 1;  // (q + 1) >> 1
    for (int w = 0; w < l; ++w) {
        const u64 s = prod[w] + carry;
        carry = (carry && s == 0) ? 1 : 0;
        half[w] = s;
    }
    for (int w = 0; w < l; ++w) half[w] = (half[w] >> 1) | (w + 1 < l ? half[w + 1] << 63 : (u64)carry << 63);
    return big;
}

}  // namespace

namespace hecuda {
namespace api {

size_t decrypt_scratch_words(const Context &c, int polys, int l) { return ((size_t)polys * l + l) * c.n; }

cudaError_t decrypt_device(const Context &c, const u64 *d_sk, const u64 *d_ct, int polys, int l, u64 *scratch, u64 *out,
                           int64_t items, cudaStream_t s) {
    return decrypt_chunk(c, make_consts(c, l, 1), scratch, d_sk, d_ct, polys, out, items, s);
}

}  // namespace api
}  // namespace hecuda

extern "C" {

int32_t hecuda_bfv_decrypt(const hecuda_context *h, const uint64_t *secret_key, const uint64_t *ciphertexts, int32_t polys,
                           int32_t l, uint64_t scaling_factor, uint64_t *plaintexts, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!secret_key) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (polys < 2 || polys > 3) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count must be 2 or 3");
    if (l < 1 || l > c.L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (batch < 0 || (batch && (!ciphertexts || !plaintexts))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    if (c.t >= c.gamma) return fail(HECUDA_ERR_UNSUPPORTED, "plaintext modulus too large");
    if (batch == 0) return HECUDA_OK;
    const DecryptConsts dc = make_consts(c, l, scaling_factor);
    // SecretKey.poly has K = L + 1 rows (Eval); rows 0..l-1 are the ones a level-l ciphertext uses
    u64 *d_sk = nullptr;
    CK(cudaMalloc(&d_sk, (size_t)l * c.n * sizeof(u64)));
    cudaError_t e = upload(d_sk, secret_key, (size_t)l * c.n * sizeof(u64));
    if (e != cudaSuccess) {
        cudaFree(d_sk);
        return cuda_fail(e, "secret key upload");
    }
    const size_t in_words = (size_t)polys * l * c.n;
    const int64_t chunk = std::max<int64_t>(1, (int64_t)((size_t)64 * 1024 * 1024 / in_words));
    WsGuard g(h);
    if (!g.w) {
        cudaFree(d_sk);
        return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    }
    cudaStream_t s = g.w->stream;
    u64 *d_in = nullptr, *d_scratch = nullptr, *d_out = nullptr;
    const int64_t cap = std::min<int64_t>(chunk, batch);
    e = cudaMallocAsync((void **)&d_in, in_words * cap * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_scratch, (in_words + (size_t)l * c.n) * cap * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_out, (size_t)c.n * cap * sizeof(u64), s);
    for (int64_t done = 0; e == cudaSuccess && done < batch; done += cap) {
        const int64_t items = std::min<int64_t>(cap, batch - done);
        e = cudaMemcpyAsync(d_in, ciphertexts + in_words * done, in_words * items * sizeof(u64), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = decrypt_chunk(c, dc, d_scratch, d_sk, d_in, polys, d_out, items, s);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(plaintexts + (size_t)c.n * done, d_out, (size_t)c.n * items * sizeof(u64), cudaMemcpyDeviceToHost, s);
    }
    if (d_in) cudaFreeAsync(d_in, s);
    if (d_scratch) cudaFreeAsync(d_scratch, s);
    if (d_out) cudaFreeAsync(d_out, s);
    cudaError_t e2 = cudaStreamSynchronize(s);
    fill(d_sk, 0, (size_t)l * c.n * sizeof(u64));  // zeroize the key copy (the reference zeroizes SecretKey storage)
    cudaFree(d_sk);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "decrypt");
}

int32_t hecuda_bfv_noise_budget(const hecuda_context *h, const uint64_t *secret_key, const uint64_t *ciphertexts, int32_t polys,
                                int32_t l, int32_t eval_format, double *budgets, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    const Context &c = *h->ctx;
    if (!secret_key) return fail(HECUDA_ERR_MISSING_KEY, "null secret key");
    if (polys < 2 || polys > 3) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: poly_count must be 2 or 3");
    if (l < 1 || l > c.L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: moduli_count out of range");
    if (batch < 0 || (batch && (!ciphertexts || !budgets))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    if (batch == 0) return HECUDA_OK;
    const DecryptConsts dc = make_consts(c, l, 1);
    NoiseConsts nc;
    nc.l = l;
    for (int i = 0; i < l; ++i) {
        nc.q[i] = dc.q[i];
        nc.t_mod[i] = c.t % dc.q[i];
        nc.inv_punctured[i] = dc.inv_punctured[i];
    }
    const std::vector<u64> big = noise_big_constants(dc.q, l);
    const int64_t n = c.n;
    const size_t in_words = (size_t)polys * l * n;
    const int64_t cap = std::min<int64_t>(batch, std::max<int64_t>(1, (int64_t)((size_t)64 * 1024 * 1024 / in_words)));
    std::vector<u64> norms((size_t)batch * l);
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    u64 *d_sk = nullptr, *d_big = nullptr, *d_in = nullptr, *d_ev = nullptr, *d_dot = nullptr, *d_norm = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_sk, (size_t)l * n * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_big, big.size() * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_in, in_words * cap * sizeof(u64), s);
    if (e == cudaSuccess && !eval_format) e = cudaMallocAsync((void **)&d_ev, in_words * cap * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_dot, (size_t)l * n * cap * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_norm, (size_t)l * cap * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_sk, secret_key, (size_t)l * n * sizeof(u64), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_big, big.data(), big.size() * sizeof(u64), cudaMemcpyHostToDevice, s);
    const NttRowMap map = c.map_q(l);
    const int threads = coeff_threads(n);
    const unsigned gx = (unsigned)((n + threads - 1) / threads);
    for (int64_t done = 0; e == cudaSuccess && done < batch; done += cap) {
        const int64_t items = std::min<int64_t>(cap, batch - done);
        e = cudaMemcpyAsync(d_in, ciphertexts + in_words * done, in_words * items * sizeof(u64), cudaMemcpyHostToDevice, s);
        const u64 *ev = d_in;
        if (e == cudaSuccess && !eval_format) {  // noiseBudgetCoeff = noiseBudgetEval of convertToEvalFormat (:181-185)
            e = launch_ntt_forward(c, map, d_in, d_ev, items * polys * l, s);
            ev = d_ev;
        }
        if (e == cudaSuccess)
            e = for_each_part(items, [&](int64_t first, int64_t part) {
                return launch(dot_secret_kernel, dim3(gx, (unsigned)l, (unsigned)part), threads, 0, s,
                              ev + first * polys * l * n, d_sk, d_dot + first * l * n, dc, (int)n, polys);
            });
        if (e == cudaSuccess) e = launch_ntt_inverse(c, map, d_dot, d_dot, items * l, kScalePlain, s);
        if (e == cudaSuccess) e = launch(noise_norm_kernel, (unsigned)items, kNormThreads, 0, s, d_dot, d_big, nc, (int)n, d_norm);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(norms.data() + (size_t)l * done, d_norm, (size_t)l * items * sizeof(u64), cudaMemcpyDeviceToHost, s);
    }
    if (d_sk) cudaMemsetAsync(d_sk, 0, (size_t)l * n * sizeof(u64), s);  // zeroize the key copy
    if (d_dot) cudaMemsetAsync(d_dot, 0, (size_t)l * n * cap * sizeof(u64), s);  // v = m Delta + noise: secret too
    for (void *p : {(void *)d_sk, (void *)d_big, (void *)d_in, (void *)d_ev, (void *)d_dot, (void *)d_norm})
        if (p) cudaFreeAsync(p, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    if (e != cudaSuccess) return cuda_fail(e, "noise_budget");
    double q_double = 1.0;  // vTimesT.moduli.map { Double($0) }.reduce(1.0, *)
    for (int i = 0; i < l; ++i) q_double *= (double)dc.q[i];
    for (int64_t b = 0; b < batch; ++b) {
        const double norm = host::wide_to_double(norms.data() + (size_t)l * b, l);
        budgets[b] = norm == 0.0 ? HUGE_VAL : std::log2(q_double / (2 * norm));
    }
    return HECUDA_OK;
}

}  // extern "C"
