// drbg.cu -- seeded-ciphertext expansion on the device (SURVEY.md 8f rank 4).
//
//   NistCtrDrbg (CTR_DRBG, AES-128, no derivation function)   Random/NistCtrDrbg.swift:25-84  (NIST SP 800-90A)
//   NistAes128Ctr = BufferedRng<NistCtrDrbg>, 4096-byte buffer Random/NistAes128Ctr.swift:17-40, BufferedRng.swift:17-67
//   PolyRq.randomizeUniform(using:)                            PolyRq/PolyRq+Randomize.swift:49-81
//   Ciphertext(deserialize: .seeded(poly0:seed:))              SerializedCiphertext.swift:41-60
//
// The byte stream a seed produces is a chain of 4096-byte segments: segment s is AES-128-CTR under (key_s, V_s), and
// (key_{s+1}, V_{s+1}) come from two more blocks of the same keystream.  One thread per seed walks that chain (it is
// inherently sequential, 2 block encryptions + 1 key schedule per segment) and leaves the expanded round keys; then
// every 16-byte block of every segment is independent: one CTA per segment, one thread per block = per coefficient
// (a coefficient consumes exactly one little-endian 128-bit word, reduced modulo its row modulus).  Seeded evaluation
// keys (EvaluationKey(deserialize:), SerializedKeys.swift:141-157) use the same chain over K = L + 1 rows, then one fused
// kernel that also unpacks poly0 and writes both polys into the key buffers.
// AES is FIPS-197 written from the specification (S-box, ShiftRows, MixColumns over GF(2^8)); the reference gets it
// from swift-crypto.  Pinned by the reference's NIST vectors through the oracle (tests/test_oracle_drbg.py).
#include "capi_internal.hpp"
#include "drbg.cuh"
#include "modarith.cuh"
#include "simple_pir.cuh"

using namespace hecuda;
using namespace hecuda::api;
using namespace hecuda::drbg;

namespace {

__constant__ unsigned char c_sbox[256];
__constant__ u32w c_te0[256];

__device__ __forceinline__ void load_tables(unsigned char *sbox, u32w *te0) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        sbox[i] = c_sbox[i];
        te0[i] = c_te0[i];
    }
    __syncthreads();
}

// The 128-bit word of this thread's block (counter V + 1 + threadIdx.x) of a segment whose (V hi, V lo) is at ctr:
// UInt128(littleEndianBytes:) of the 16 output bytes, byte i of the block being bits 8i.. of the value
__device__ __forceinline__ u128 segment_word(const u32w *rk, const u64 *ctr, const u32w *te0, const unsigned char *sbox) {
    u32w blk[4];
    counter_block(ctr[0], ctr[1], 1 + (u64)threadIdx.x, blk);
    encrypt_block(blk, rk, te0, sbox);
    const u64 lo = (u64)__byte_perm(blk[0], 0, 0x0123) | ((u64)__byte_perm(blk[1], 0, 0x0123) << 32);
    const u64 hi = (u64)__byte_perm(blk[2], 0, 0x0123) | ((u64)__byte_perm(blk[3], 0, 0x0123) << 32);
    return ((u128)hi << 64) | lo;
}

// two lanes per seed walk its chain of segments: both expand the current key, lane p encrypts counter block V + 1 + p,
// the pair exchanges the blocks by shuffle and absorbs them (ctrDrbgUpdate); lane 0 leaves (round keys, V) of each segment.
// Seed b is the 32 bytes at seeds + seed_at[b] (seeds read in place from a message), or at seeds + 32 b without seed_at.
__global__ void __launch_bounds__(64) drbg_chain_kernel(const unsigned char *__restrict__ seeds,
                                                        const long long *__restrict__ seed_at, u32w *__restrict__ round_keys,
                                                        u64 *__restrict__ counters, int segments, long long batch) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(sbox, te0);
    const long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 1;
    const int lane = threadIdx.x & 1;
    const bool live = b < batch;  // dead pairs still take part in the shuffles
    const long long seed = live ? b : 0;
    u32w key[4] = {0, 0, 0, 0}, rk[kRoundKeyWords], blk[4], b0[4], b1[4], provided[8];
    u64 hi = 0, lo = 0;
    for (int i = 0; i < 8; ++i) {
        const unsigned char *p = seeds + (seed_at ? seed_at[seed] : 32 * seed) + 4 * i;
        provided[i] = ((u32w)p[0] << 24) | ((u32w)p[1] << 16) | ((u32w)p[2] << 8) | p[3];
    }
    for (int s = -1; s < segments; ++s) {  // s = -1: init(entropy:) (NistCtrDrbg.swift:52-59)
        expand_key(key, rk, sbox);
        if (s >= 0) {
            if (live && lane == 0) {
                u32w *dst = round_keys + ((size_t)b * segments + s) * kRoundKeyWords;
                for (int i = 0; i < kRoundKeyWords; ++i) dst[i] = rk[i];
                counters[2 * ((size_t)b * segments + s)] = hi;
                counters[2 * ((size_t)b * segments + s) + 1] = lo;
            }
            const u64 l = lo + kSegmentBlocks;  // ctrDrbgGenerate(count: 4096) advances V by 256 blocks (:71-84)
            hi += l < lo ? 1 : 0;
            lo = l;
        }
        counter_block(hi, lo, 1 + (u64)lane, blk);
        encrypt_block(blk, rk, te0, sbox);
        for (int i = 0; i < 4; ++i) {
            b0[i] = __shfl_sync(0xffffffffu, blk[i], (threadIdx.x & 30), 32);
            b1[i] = __shfl_sync(0xffffffffu, blk[i], (threadIdx.x & 30) | 1, 32);
        }
        drbg_absorb(key, hi, lo, b0, b1, s < 0 ? provided : nullptr);
    }
}

// one CTA per segment, one thread per 16-byte block = per coefficient (randomizeUniform, PolyRq+Randomize.swift:58-80)
__global__ void __launch_bounds__(kSegmentBlocks) drbg_fill_kernel(const u32w *__restrict__ round_keys,
                                                                   const u64 *__restrict__ counters, u64 *__restrict__ out,
                                                                   const __grid_constant__ RowModuli c, int n, int segments) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    __shared__ u32w rk[kRoundKeyWords];
    const long long b = blockIdx.y;
    const int s = blockIdx.x;
    if (threadIdx.x < kRoundKeyWords) rk[threadIdx.x] = round_keys[((size_t)b * segments + s) * kRoundKeyWords + threadIdx.x];
    load_tables(sbox, te0);
    const long long k = (long long)s * kSegmentBlocks + threadIdx.x;
    if (k >= (long long)c.rows * n) return;
    const int row = (int)(k / n);
    out[(size_t)b * c.rows * n + k] = (u64)(segment_word(rk, counters + 2 * ((size_t)b * segments + s), te0, sbox) % c.p[row]);
}

// PolyRq.random over one modulus for `total` = polys x N coefficients of one stream (SimplePirContext
// .generateAPolynomials, SimplePir+Database.swift:181-184), stored as a, or as sigma(a) = a(x^-1) (simple_pir.cuh)
__global__ void __launch_bounds__(kSegmentBlocks) drbg_one_modulus_fill_kernel(const u32w *__restrict__ round_keys,
                                                                               const u64 *__restrict__ counters,
                                                                               u64 *__restrict__ out, u64 p, long long n,
                                                                               long long total, bool sigma) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    __shared__ u32w rk[kRoundKeyWords];
    const int s = blockIdx.x;
    if (threadIdx.x < kRoundKeyWords) rk[threadIdx.x] = round_keys[(size_t)s * kRoundKeyWords + threadIdx.x];
    load_tables(sbox, te0);
    const long long k = (long long)s * kSegmentBlocks + threadIdx.x;
    if (k >= total) return;
    const u64 v = (u64)(segment_word(rk, counters + 2 * (size_t)s, te0, sbox) % p);
    const long long poly = k / n, i = k - poly * n;
    if (sigma)
        out[poly * n + spir::sigma_index(i, n)] = spir::sigma_value(v, i, p);
    else
        out[k] = v;
}

// EvaluationKey(deserialize:) of seeded key-switching ciphertexts (SerializedCiphertext.swift:53-60 with Format = Eval):
// one CTA per (segment, ciphertext), one thread per coefficient k of the K x N stream.  poly1 = the DRBG word reduced
// modulo its row's modulus, already in the key's Eval format (encryptZero samples `a` in Eval, Bfv+Encrypt.swift:156-157,
// and convertFormat to Eval is the identity); poly0 = coefficient k unpacked from the ciphertext's serialized bytes.
// Both go straight into the ciphertext's 2 x K x N words at dst[ciphertext].  Ciphertext b's poly0 is at
// poly0 + b x byteCount, or, with at.tag, at poly0 + at.tag[at.first + b] - at.base (read in place from a message).
__global__ void __launch_bounds__(kSegmentBlocks) key_expand_kernel(const u32w *__restrict__ round_keys,
                                                                    const u64 *__restrict__ counters,
                                                                    const unsigned char *__restrict__ poly0,
                                                                    u64 *const *__restrict__ dst, const __grid_constant__ RowModuli c,
                                                                    const __grid_constant__ CodecConsts cc, int n, int segments,
                                                                    const __grid_constant__ PolyLayout at) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    __shared__ u32w rk[kRoundKeyWords];
    const long long b = blockIdx.y;
    const int s = blockIdx.x;
    if (threadIdx.x < kRoundKeyWords) rk[threadIdx.x] = round_keys[((size_t)b * segments + s) * kRoundKeyWords + threadIdx.x];
    load_tables(sbox, te0);
    const long long k = (long long)s * kSegmentBlocks + threadIdx.x;
    if (k >= (long long)c.rows * n) return;
    const u128 word = segment_word(rk, counters + 2 * ((size_t)b * segments + s), te0, sbox);
    const int row = (int)(k / n);
    const long long i = k - (long long)row * n;
    const unsigned char *src =
        poly0 + (at.tag ? at.tag[at.first + b] - at.base : b * cc.byte_offset[cc.rows]) + cc.byte_offset[row];
    u64 *out = dst[b];
    out[k] = codec_unpack(src, cc.byte_offset[row + 1] - cc.byte_offset[row], cc.width[row], i);
    out[(long long)c.rows * n + k] = (u64)(word % c.p[row]);
}

}  // namespace

namespace hecuda {
namespace api {

// The AES tables, then every seed's chain: (round keys, V) of each of its `segments` segments into *d_rk / *d_ctr, both
// allocated on `s` and released by free_chains.
cudaError_t drbg_upload_tables(cudaStream_t s) {
    unsigned char sbox[256];
    u32w te0[256];
    make_tables(sbox, te0);
    cudaError_t e = cudaMemcpyToSymbolAsync(c_sbox, sbox, sizeof(sbox), 0, cudaMemcpyHostToDevice, s);  // per device, cheap
    if (e == cudaSuccess) e = cudaMemcpyToSymbolAsync(c_te0, te0, sizeof(te0), 0, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(s);  // the tables live on this stack frame
}

cudaError_t drbg_chains(const unsigned char *d_seeds, int segments, int64_t batch, u32w **d_rk, u64 **d_ctr, cudaStream_t s,
                        const long long *d_seed_at) {
    const cudaError_t e = drbg_upload_tables(s);
    return e == cudaSuccess ? drbg_chains_uploaded(d_seeds, segments, batch, d_rk, d_ctr, s, d_seed_at) : e;
}

cudaError_t drbg_chains_uploaded(const unsigned char *d_seeds, int segments, int64_t batch, u32w **d_rk, u64 **d_ctr,
                                 cudaStream_t s, const long long *d_seed_at) {
    cudaError_t e = cudaMallocAsync((void **)d_rk, (size_t)batch * segments * kRoundKeyWords * sizeof(u32w), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)d_ctr, (size_t)batch * segments * 2 * sizeof(u64), s);
    if (e == cudaSuccess) e = launch(drbg_chain_kernel, (unsigned)((batch + 31) / 32), 64, 0, s, d_seeds, d_seed_at, *d_rk, *d_ctr, segments, batch);
    return e;
}

void free_chains(u32w *d_rk, u64 *d_ctr, int segments, int64_t batch, cudaStream_t s) {
    if (d_rk) {
        cudaMemsetAsync(d_rk, 0, (size_t)batch * segments * kRoundKeyWords * sizeof(u32w), s);  // key material
        cudaFreeAsync(d_rk, s);
    }
    if (d_ctr) cudaFreeAsync(d_ctr, s);
}

// PolyRq.random mod p for `polys` polynomials of degree n from the one NistAes128Ctr stream of the 32-byte d_seed,
// written as a (sigma false) or sigma(a) (drbg_one_modulus_fill_kernel) to d_out (polys x n)
cudaError_t random_polys_one_modulus_device(const unsigned char *d_seed, u64 p, int64_t n, int64_t polys, bool sigma,
                                            u64 *d_out, cudaStream_t s) {
    const int64_t total = polys * n;
    const int segments = (int)((total * 16 + kSegmentBytes - 1) / kSegmentBytes);
    u32w *d_rk = nullptr;
    u64 *d_ctr = nullptr;
    cudaError_t e = drbg_chains(d_seed, segments, 1, &d_rk, &d_ctr, s);
    if (e == cudaSuccess)
        e = launch(drbg_one_modulus_fill_kernel, (unsigned)segments, kSegmentBlocks, 0, s, d_rk, d_ctr, d_out, p,
                   (long long)n, (long long)total, sigma);
    free_chains(d_rk, d_ctr, segments, 1, s);
    return e;
}

cudaError_t random_sigma_polys_device(const unsigned char *d_seed, u64 p, int64_t n, int64_t polys, u64 *d_out,
                                      cudaStream_t s) {
    return random_polys_one_modulus_device(d_seed, p, n, polys, true, d_out, s);
}

// Device addresses of the AES tables drbg_chains uploads, for kernels in other translation units that read a stream
cudaError_t drbg_tables(const unsigned char **sbox, const u32w **te0) {
    cudaError_t e = cudaGetSymbolAddress((void **)sbox, c_sbox);
    return e == cudaSuccess ? cudaGetSymbolAddress((void **)te0, c_te0) : e;
}

}  // namespace api
}  // namespace hecuda

namespace {

cudaError_t random_polys_device(const Context &c, int l, const unsigned char *d_seeds, u64 *d_out, int64_t batch,
                                cudaStream_t s, const long long *d_seed_at = nullptr) {
    const int segments = (int)(((size_t)l * c.n * 16 + kSegmentBytes - 1) / kSegmentBytes);
    u32w *d_rk = nullptr;
    u64 *d_ctr = nullptr;
    cudaError_t e = drbg_chains(d_seeds, segments, batch, &d_rk, &d_ctr, s, d_seed_at);
    const RowModuli fc = row_moduli(c, c.map_q(l));
    if (e == cudaSuccess)
        e = for_each_part(batch, [&](int64_t done, int64_t part) {
            return launch(drbg_fill_kernel, dim3((unsigned)segments, (unsigned)part), kSegmentBlocks, 0, s,
                          d_rk + (size_t)done * segments * kRoundKeyWords, d_ctr + (size_t)done * segments * 2,
                          d_out + (size_t)done * l * c.n, fc, (int)c.n, segments);
        });
    free_chains(d_rk, d_ctr, segments, batch, s);
    return e;
}

int32_t check(const hecuda_context *h, const void *seeds, int32_t l, const void *out, int64_t batch) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (l < 1 || l > h->ctx->L) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidPolyContext: moduli_count out of range");
    if (batch < 0 || (batch && (!seeds || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    return HECUDA_OK;
}

}  // namespace

namespace hecuda {
namespace api {

// Ciphertext(deserialize: .seeded) for `batch` ciphertexts, all buffers on the device; d_out: batch x 2 x l x N (Coeff).
// Contiguous: d_poly0 holds batch x byteCount(l rows) bytes and d_seeds batch x 32.  With at.tag, both are read in place
// from the bytes at d_poly0 (d_seeds unused): ciphertext b's poly0 at at.tag[b] (frame 0: zero rows where tag[b + 1] ==
// tag[b]) and its seed at at.seed[b].
cudaError_t expand_seeded_device(const Context &c, int l, const unsigned char *d_poly0, const unsigned char *d_seeds, u64 *d_out,
                                 int64_t batch, cudaStream_t s, const PolyLayout &at) {
    const NttRowMap map = c.map_q(l);
    CodecConsts cc;
    std::string err;
    if (!codec_consts(c, map, 0, cc, err)) return cudaErrorInvalidValue;
    const size_t poly_words = (size_t)l * c.n, pw = poly_words * sizeof(u64);
    u64 *d_a = nullptr, *d_p0 = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_a, pw * batch, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_p0, pw * batch, s);
    // poly0: PolyRq(deserialize:) ; poly1: random Eval polynomial converted to Coeff (SerializedCiphertext.swift:44-49)
    if (e == cudaSuccess) e = launch_poly_load(c, cc, 0, d_poly0, d_p0, batch, s, at);
    if (e == cudaSuccess) e = at.tag ? random_polys_device(c, l, d_poly0, d_a, batch, s, at.seed)
                                     : random_polys_device(c, l, d_seeds, d_a, batch, s);
    if (e == cudaSuccess) e = launch_ntt_inverse(c, map, d_a, d_a, batch * l, kScalePlain, s);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(d_out, 2 * pw, d_p0, pw, pw, (size_t)batch, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(d_out + poly_words, 2 * pw, d_a, pw, pw, (size_t)batch, cudaMemcpyDeviceToDevice, s);
    if (d_a) cudaFreeAsync(d_a, s);
    if (d_p0) cudaFreeAsync(d_p0, s);
    return e;
}

int key_segments(const Context &c) {
    return (int)(((size_t)(c.L + 1) * c.n * 16 + kSegmentBytes - 1) / kSegmentBytes);
}

cudaError_t expand_key_ciphertexts(const Context &c, const u32w *d_rk, const u64 *d_ctr, int64_t first, int64_t count,
                                   const unsigned char *d_poly0, u64 *const *d_dst, cudaStream_t s, const PolyLayout &layout) {
    const NttRowMap map = c.map_ks(c.L);  // row K-1 is q_ks
    CodecConsts cc;
    std::string err;
    if (!codec_consts(c, map, 0, cc, err)) return cudaErrorInvalidValue;
    const int segments = key_segments(c);
    const RowModuli fc = row_moduli(c, map);
    return for_each_part(count, [&](int64_t done, int64_t part) {
        const size_t at = (size_t)(first + done) * segments;
        PolyLayout from = layout;
        from.first += done;
        return launch(key_expand_kernel, dim3((unsigned)segments, (unsigned)part), kSegmentBlocks, 0, s,
                      d_rk + at * kRoundKeyWords, d_ctr + at * 2,
                      d_poly0 + (layout.tag ? 0 : (size_t)done * serialized_poly_bytes(cc)), d_dst + first + done, fc, cc,
                      (int)c.n, segments, from);
    });
}

}  // namespace api
}  // namespace hecuda

extern "C" {

int32_t hecuda_poly_random_from_seed(const hecuda_context *h, const uint8_t *seeds, int32_t l, uint64_t *out, int64_t batch) {
    int32_t rc = check(h, seeds, l, out, batch);
    if (rc || batch == 0) return rc;
    const Context &c = *h->ctx;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    unsigned char *d_seeds = nullptr;
    u64 *d_out = nullptr;
    const size_t words = (size_t)l * c.n * batch;
    cudaError_t e = cudaMallocAsync((void **)&d_seeds, (size_t)32 * batch, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_out, words * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seeds, seeds, (size_t)32 * batch, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = random_polys_device(c, l, d_seeds, d_out, batch, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, words * sizeof(u64), cudaMemcpyDeviceToHost, s);
    if (d_seeds) cudaFreeAsync(d_seeds, s);
    if (d_out) cudaFreeAsync(d_out, s);
    cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "poly_random_from_seed");
}

int32_t hecuda_ciphertext_expand_seeded(const hecuda_context *h, const uint8_t *poly0, const uint8_t *seeds, int32_t l,
                                        uint64_t *out, int64_t batch) {
    int32_t rc = check(h, seeds, l, out, batch);
    if (rc) return rc;
    if (batch && !poly0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    if (batch == 0) return HECUDA_OK;
    const Context &c = *h->ctx;
    const NttRowMap map = c.map_q(l);
    CodecConsts cc;
    std::string err;
    if (!codec_consts(c, map, 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const size_t poly_bytes = (size_t)serialized_poly_bytes(cc), poly_words = (size_t)l * c.n;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    unsigned char *d_seeds = nullptr, *d_poly0 = nullptr;
    u64 *d_out = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_seeds, (size_t)32 * batch, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_poly0, poly_bytes * batch, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_out, 2 * poly_words * batch * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seeds, seeds, (size_t)32 * batch, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_poly0, poly0, poly_bytes * batch, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = expand_seeded_device(c, l, d_poly0, d_seeds, d_out, batch, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, 2 * poly_words * sizeof(u64) * batch, cudaMemcpyDeviceToHost, s);
    for (void *p : {(void *)d_seeds, (void *)d_poly0, (void *)d_out})
        if (p) cudaFreeAsync(p, s);
    cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "expand_seeded");
}

}  // extern "C"
