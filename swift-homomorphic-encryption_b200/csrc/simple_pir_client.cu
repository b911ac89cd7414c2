// simple_pir_client.cu -- SimplePIR's client on the device: batched query precompute (secrets, noiselessSample through
// the NTT, modSwitch, error, deltas) with resultsWithoutResponse = S . hint^T mod p on the integer tensor cores, and
// batched decryption.  The arithmetic and index maps are in simple_pir.cuh.
//
//   DefaultQueryGenerator.init (generateAPolynomials, convertToEvalFormat)   SimplePir+Precompute.swift:328-334
//   PrecomputedQueries.WithoutIndices.init, add(index:)                      SimplePir+Precompute.swift:199-256
//   generateSecretPolys, noiselessSample, encryptZero, extractEntries        SimplePir+Client.swift:20-95
//   WithPreparedResponse.integrate, SimplePirClient.decrypt                  SimplePir+Precompute.swift:299-311,
//                                                                            SimplePir+Client.swift:111-121
//
// A precompute of `count` queries (Q = count x chunksPerEntry secret rows):
//   1. the DRBG chains of the secret and error seeds (drbg.cu; the AES tables are uploaded by _create);
//   2. ternary_kernel: every secret coefficient, as a u64 row mod p and as the [s = 1] / [s = -1] u8 masks in the
//      mma.m16n8k32 B-operand layout;
//   3. forward NTT of the Q rows;
//   4. per slab of rows: the pointwise products with every NTT(a_j), one inverse NTT, and finish_kernel
//      (divideAndRound, the error, the delta) into the query words;
//   5. results_kernel: per (hint plane, mask) an MMA chain over N, then the reference's wrapping double-width sum mod p.
// Every device copy of the secrets (rows, their NTTs, the products, the masks, the seeds) is zeroized before it is freed.
#include <algorithm>
#include <initializer_list>
#include <vector>

#include "capi_internal.hpp"
#include "sampling.cuh"
#include "simple_pir.cuh"

using namespace hecuda;
using namespace hecuda::api;
using namespace hecuda::drbg;

struct hecuda_simple_pir_client {
    int device = 0;
    hecuda_simple_pir_params params{};
    int64_t m = 0, k = 0, n = 0, blocks = 0;  // hint M x N; K query columns; aPolyCount
    int64_t entry_scalars = 0, chunk = 0;     // chunkSize
    u64 p = 0, mu_hi = 0, mu_lo = 0;          // nttFriendlyMod, floor(2^128 / p)
    hecuda::Context *ctx = nullptr;           // the single-modulus extraContext
    u64 *d_a = nullptr;                       // NTT(a_j): blocks x N
    unsigned char *d_hint = nullptr;          // hint digit planes (simple_pir.cuh, a_offset)
    int planes = 0;                           // ceil((ct + 1) / 8)
    int64_t row_tiles = 0, col_tiles = 0;
    size_t plane_bytes = 0;
    const unsigned char *sbox = nullptr;      // the AES tables on the device (drbg.cu)
    const u32w *te0 = nullptr;
    int cbd_words = 0;
    u64 cbd_mask = 0;
};

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = 4, kWarpRowTiles = 2, kCtaQueryTiles = 2;  // results_kernel: as simple_pir.cu's response kernel
constexpr int kCtaRows = kWarps * kWarpRowTiles * spir::kTileRows, kCtaQueries = kCtaQueryTiles * spir::kTileQueries;
constexpr int64_t kSlabWords = 32ll << 20;  // <= 256 MB of noiselessSample rows per slab

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

// the hint (M x N words < p) into its digit planes; thread (row, four columns) of the padded plane
template <typename W>
__global__ void __launch_bounds__(kThreads) hint_pack_kernel(const W *__restrict__ hint, long long m, long long n,
                                                             long long rows_pad, long long col_tiles, int planes,
                                                             size_t plane_bytes, unsigned char *__restrict__ out) {
    const long long quads = col_tiles * (spir::kTileCols / 4);
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows_pad * quads) return;
    const long long c0 = t % quads * 4, r = t / quads;
    u64 v[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) v[b] = r < m && c0 + b < n ? (u64)hint[r * n + c0 + b] : 0;
    const long long at = spir::a_offset(r, c0, col_tiles);
    for (int d = 0; d < planes; ++d) {
        unsigned w = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) w |= spir::db_digit(v[b], d) << (8 * b);
        *reinterpret_cast<unsigned *>(out + d * plane_bytes + at) = w;
    }
}

// generateSecretPolys for secret row r = r0 + blockIdx.y (query r / cpe, polynomial r % cpe), coefficient j: the row
// mod p (-1 as p - 1) and the two masks at b_offset(r, j)
__global__ void __launch_bounds__(kThreads) ternary_kernel(const u32w *__restrict__ rk, const u64 *__restrict__ ctr,
                                                           int segments, const __grid_constant__ Tables g, u64 p, int n,
                                                           int cpe, long long col_tiles, u64 *__restrict__ rows,
                                                           unsigned char *__restrict__ masks, long long mask_bytes,
                                                           long long r0) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long r = r0 + blockIdx.y;
    StreamReader st = reader(rk, ctr, segments, r / cpe, sbox, te0);
    const u64 v = ternary_value(st, spir::secret_coefficient(r % cpe, j, n));
    rows[r * n + j] = signed_residue((long long)v - 1, p);
    const long long at = spir::b_offset(r, j, col_tiles);
    masks[at] = v == 2 ? 1 : 0;
    masks[mask_bytes + at] = v == 0 ? 1 : 0;
}

// noiselessSample's products in Eval: out[(rl x blocks + j) x N + c] = NTT(s)[r0 + rl][c] . NTT(a_j)[c] mod p
__global__ void __launch_bounds__(kThreads) pointwise_kernel(const u64 *__restrict__ s_hat, const u64 *__restrict__ a_hat,
                                                             long long r0, long long rows, long long blocks, long long n,
                                                             u64 p, u64 mu_hi, u64 mu_lo, u64 *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows * blocks * n) return;
    const long long c = t % n, jb = t / n % blocks, rl = t / n / blocks;
    const u64 x = s_hat[(r0 + rl) * n + c], y = a_hat[jb * n + c];
    uint64_t rem;
    spir::div_mod((spir::spir_u128)x * y, p, mu_hi, mu_lo, rem);
    out[t] = rem;
}

struct FinishArgs {
    u64 p, mu_hi, mu_lo;
    long long k, row_words;  // K, blocks x N
    int cpe, epc, ct, pt, cbd_words;
    u64 cbd_mask;
};

// encryptZero after noiselessSample, then add(index:): thread (slab row rl, column c < K)
template <typename W>
__global__ void __launch_bounds__(kThreads) finish_kernel(const u64 *__restrict__ sample, const u32w *__restrict__ rk,
                                                          const u64 *__restrict__ ctr, int segments,
                                                          const __grid_constant__ Tables g, const FinishArgs a,
                                                          const int64_t *__restrict__ indices, long long r0, long long rows,
                                                          W *__restrict__ queries) {
    __shared__ unsigned char sbox[256];
    __shared__ u32w te0[256];
    load_tables(g, sbox, te0);
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows * a.k) return;
    const long long rl = t / a.k, c = t - rl * a.k, r = r0 + rl, q = r / a.cpe, i = r - q * a.cpe;
    const u64 mask = spir::low_mask(a.ct);
    u64 v = spir::divide_and_round(sample[rl * a.row_words + c], a.p, a.mu_hi, a.mu_lo, a.ct);
    StreamReader st = reader(rk, ctr, segments, q, sbox, te0);
    const int e = cbd_value(st, spir::error_coefficient(i, c, a.k), a.cbd_words, a.cbd_mask);
    v = (v + (signed_residue(e, 1ull << a.ct) & mask)) & mask;
    if (indices && c == spir::delta_column(indices[q], i, a.cpe, a.epc)) v = (v + (1ull << (a.ct - a.pt))) & mask;
    queries[r * a.k + c] = (W)v;
}

struct ResultsArgs {
    const unsigned char *hint;
    size_t plane_bytes;
    int planes, word_bits;
    long long col_tiles, m, q;
    const unsigned char *masks;  // [s = 1], then [s = -1]
    long long mask_bytes;
    u64 p, mu_hi, mu_lo;
};

// resultsWithoutResponse: warp w owns hint row tiles (blockIdx.x x kWarps + w) x 2 + {0, 1} and secret-row tiles
// qt_first + blockIdx.y x 2 + {0, 1}; per hint plane d, the MMA chains of both masks over N give P_d and Nn_d (each
// < 2^15 x 255, no slicing), added into the wrapping 128-bit sum; out[row_q][row] = U mod p
template <typename W>
__global__ void __launch_bounds__(kWarps * 32) results_kernel(const ResultsArgs a, long long qt_first, W *__restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long rt0 = ((long long)blockIdx.x * kWarps + warp) * kWarpRowTiles;
    if (rt0 * spir::kTileRows >= a.m) return;  // padding rows only; no block-wide barrier
    const long long qt0 = qt_first + (long long)blockIdx.y * kCtaQueryTiles;
    spir::spir_u128 acc[kWarpRowTiles][kCtaQueryTiles][4];
#pragma unroll
    for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
        for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0;
    for (int d = 0; d < a.planes; ++d) {
        int sum[2][kWarpRowTiles][kCtaQueryTiles][4];
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
                for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) sum[b][mt][nt][e] = 0;
        const uint4 *pa = reinterpret_cast<const uint4 *>(a.hint + d * a.plane_bytes) + rt0 * a.col_tiles * 32 + lane;
        for (long long kt = 0; kt < a.col_tiles; ++kt) {
            uint4 fa[kWarpRowTiles];
#pragma unroll
            for (int mt = 0; mt < kWarpRowTiles; ++mt) fa[mt] = __ldg(pa + (mt * a.col_tiles + kt) * 32);
#pragma unroll
            for (int b = 0; b < 2; ++b) {
                const uint2 *pb = reinterpret_cast<const uint2 *>(a.masks + b * a.mask_bytes) + lane;
#pragma unroll
                for (int nt = 0; nt < kCtaQueryTiles; ++nt) {
                    const uint2 fb = __ldg(pb + ((qt0 + nt) * a.col_tiles + kt) * 32);
#pragma unroll
                    for (int mt = 0; mt < kWarpRowTiles; ++mt) spir::mma_u8(sum[b][mt][nt], fa[mt], fb);
                }
            }
        }
#pragma unroll
        for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
            for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    acc[mt][nt][e] = spir::results_add(acc[mt][nt][e], (u32)sum[0][mt][nt][e], (u32)sum[1][mt][nt][e], d, a.p);
    }
    // C fragment: e = 0, 1 at (row g, secret rows 2t, 2t + 1), e = 2, 3 at row g + 8
    const int g = lane >> 2, tq = (lane & 3) * 2;
#pragma unroll
    for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
        for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const long long row = (rt0 + mt) * spir::kTileRows + g + (e >> 1) * 8;
                const long long query = (qt0 + nt) * spir::kTileQueries + tq + (e & 1);
                if (row < a.m && query < a.q)
                    out[query * a.m + row] = (W)spir::results_word(acc[mt][nt][e], a.word_bits, a.p, a.mu_hi, a.mu_lo);
            }
}

struct DecryptArgs {
    long long m, chunk, entry_size;
    int cpe, epc, pt, ct;
};

// integrate + coefficientsToBytes: thread (query, byte < entrySizeInBytes)
template <typename W>
__global__ void __launch_bounds__(kThreads) decrypt_kernel(const W *__restrict__ responses, const W *__restrict__ results,
                                                           const int64_t *__restrict__ indices, long long count,
                                                           const DecryptArgs a, unsigned char *__restrict__ entries) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= count * a.entry_size) return;
    const long long q = t / a.entry_size, b = t - q * a.entry_size, index = indices[q];
    const W *resp = responses + q * a.cpe * a.m, *res = results + q * a.cpe * a.m;
    entries[t] = (unsigned char)procdb::coefficients_byte(
        [&](long long c) {
            const long long at = spir::extract_offset(index, c / a.chunk, c % a.chunk, a.cpe, a.epc, a.m, a.chunk);
            return spir::integrate((u64)resp[at], (u64)res[at], a.pt, a.ct);
        },
        a.cpe * a.chunk, a.pt, b);
}

unsigned blocks_for(long long threads) { return (unsigned)((threads + kThreads - 1) / kThreads); }
int segments_for(long long bytes) { return (int)((bytes + kSegmentBytes - 1) / kSegmentBytes); }

// Device buffers of one call on one stream; the secret ones are zeroized before they are freed.
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

// The chains of `count` seeds on the device; free_chains zeroizes the round keys.
struct Streams {
    u32w *rk = nullptr;
    u64 *ctr = nullptr;
    int segments = 0;
    int64_t count = 0;
    cudaStream_t s = nullptr;
    cudaError_t make(const unsigned char *d_seeds, int segs, int64_t n, cudaStream_t st) {
        segments = segs, count = n, s = st;
        return drbg_chains_uploaded(d_seeds, segs, n, &rk, &ctr, st);
    }
    ~Streams() {
        if (s) free_chains(rk, ctr, segments, count, s);
    }
};

int64_t q_pad(int64_t rows) { return (rows + kCtaQueries - 1) / kCtaQueries * kCtaQueries; }

// WithoutIndices.init (and add(index:) with d_indices) for `count` queries already on the device, enqueued on s
template <typename W>
cudaError_t precompute_device(const hecuda_simple_pir_client &c, const unsigned char *d_secret_seeds,
                              const unsigned char *d_error_seeds, const int64_t *d_indices, int64_t count, W *d_queries,
                              W *d_results, cudaStream_t s) {
    const hecuda_simple_pir_params &pp = c.params;
    const int64_t cpe = pp.chunks_per_entry, rows = count * cpe, n = c.n;
    const long long mask_bytes = (long long)q_pad(rows) * c.col_tiles * spir::kTileCols;
    const NttRowMap map = c.ctx->map_q(1);
    const Tables tb{c.sbox, c.te0};
    cudaError_t e;
    {
        Allocs m(s);
        u64 *d_s = m.get<u64>((size_t)rows * n * sizeof(u64), true);
        unsigned char *d_masks = m.get<unsigned char>(2 * (size_t)mask_bytes, true);
        const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(rows, kSlabWords / (c.blocks * n)));
        u64 *d_prod = m.get<u64>((size_t)slab * c.blocks * n * sizeof(u64), true);
        e = m.e;
        if (e == cudaSuccess) e = cudaMemsetAsync(d_masks, 0, 2 * (size_t)mask_bytes, s);
        Streams ss, es;
        if (e == cudaSuccess) e = ss.make(d_secret_seeds, segments_for((long long)kTernaryBytes * cpe * n), count, s);
        if (e == cudaSuccess) e = es.make(d_error_seeds, segments_for(8LL * c.cbd_words * cpe * c.k), count, s);
        if (e == cudaSuccess)
            e = for_each_part(rows, [&](int64_t first, int64_t part) {
                return launch(ternary_kernel, dim3(blocks_for(n), (unsigned)part), kThreads, 0, s, ss.rk, ss.ctr, ss.segments,
                              tb, c.p, (int)n, (int)cpe, (long long)c.col_tiles, d_s, d_masks, mask_bytes, (long long)first);
            });
        if (e == cudaSuccess) e = launch_ntt_forward(*c.ctx, map, d_s, d_s, rows, s);
        const FinishArgs fa{c.p, c.mu_hi, c.mu_lo, (long long)c.k, (long long)(c.blocks * n), (int)cpe,
                            (int)pp.entries_per_column, pp.ciphertext_modulus_bits, pp.plaintext_modulus_bits, c.cbd_words,
                            c.cbd_mask};
        for (int64_t r0 = 0; e == cudaSuccess && r0 < rows; r0 += slab) {
            const int64_t part = std::min(slab, rows - r0);
            e = launch(pointwise_kernel, blocks_for(part * c.blocks * n), kThreads, 0, s, (const u64 *)d_s, (const u64 *)c.d_a,
                       (long long)r0, (long long)part, (long long)c.blocks, (long long)n, c.p, c.mu_hi, c.mu_lo, d_prod);
            if (e == cudaSuccess) e = launch_ntt_inverse(*c.ctx, map, d_prod, d_prod, part * c.blocks, kScalePlain, s);
            if (e == cudaSuccess)
                e = launch(finish_kernel<W>, blocks_for(part * c.k), kThreads, 0, s, (const u64 *)d_prod, es.rk, es.ctr,
                           es.segments, tb, fa, d_indices, (long long)r0, (long long)part, d_queries);
        }
        if (e == cudaSuccess) {
            const ResultsArgs ra{c.d_hint, c.plane_bytes, c.planes, pp.word_bits, (long long)c.col_tiles, (long long)c.m,
                                 (long long)rows, d_masks, mask_bytes, c.p, c.mu_hi, c.mu_lo};
            const unsigned gx = (unsigned)((c.m + kCtaRows - 1) / kCtaRows);
            e = for_each_part(q_pad(rows) / kCtaQueries, [&](int64_t first, int64_t part) {
                return launch(results_kernel<W>, dim3(gx, (unsigned)part), kWarps * 32, 0, s, ra,
                              (long long)(first * kCtaQueryTiles), d_results);
            });
        }
    }
    return e;
}

template <typename W>
cudaError_t decrypt_device(const hecuda_simple_pir_client &c, const W *d_responses, const W *d_results,
                           const int64_t *d_indices, int64_t count, unsigned char *d_entries, cudaStream_t s) {
    const hecuda_simple_pir_params &pp = c.params;
    const DecryptArgs a{(long long)c.m, (long long)c.chunk, (long long)pp.entry_size, (int)pp.chunks_per_entry,
                        (int)pp.entries_per_column, pp.plaintext_modulus_bits, pp.ciphertext_modulus_bits};
    return launch(decrypt_kernel<W>, blocks_for(count * pp.entry_size), kThreads, 0, s, d_responses, d_results, d_indices,
                  (long long)count, a, d_entries);
}

int32_t select_device(int device) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device available");
    if (dev != device) CK(cudaSetDevice(device));
    return HECUDA_OK;
}

// the refusals every call shares; indices (host) are checked when given
int32_t check_call(const hecuda_simple_pir_client *c, int64_t count, const int64_t *indices, bool need_indices,
                   std::initializer_list<const void *> buffers, bool host_indices) {
    if (!c) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null client");
    if (count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative query count");
    if (count == 0) return HECUDA_OK;
    for (const void *b : buffers)
        if (!b) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    if (need_indices && !indices) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null indices");
    const int64_t cpe = c->params.chunks_per_entry, epc = c->params.entries_per_column;
    if (count > (1ll << 40) / std::max<int64_t>(1, cpe * std::max(c->k, c->m)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "too many queries for one call");
    if (indices && host_indices)
        for (int64_t q = 0; q < count; ++q)  // the last chunk's column must lie inside the K columns
            if (indices[q] < 0 || indices[q] > ((c->k - 1) * epc + epc - 1 - (cpe - 1)) / cpe)
                return fail(HECUDA_ERR_INVALID_ARGUMENT, "index out of range: its query column reaches databaseColumns");
    return select_device(c->device);
}

int32_t finish_host(cudaStream_t s, cudaError_t e, const char *what) {
    if (s) {
        const cudaError_t e2 = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(s);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, what);
}

}  // namespace

extern "C" {

int32_t hecuda_simple_pir_client_create(const void *hint, const hecuda_simple_pir_params *params, const uint8_t *seed,
                                        hecuda_simple_pir_client **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    int64_t m = 0, k = 0, scalars = 0;
    u64 p = 0;
    int32_t rc = simple_pir_derive(params, m, k, scalars, p);
    if (rc) return rc;
    if (!hint || !seed) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const hecuda_simple_pir_params &pp = *params;
    const int64_t n = pp.lattice_dimension;
    const bool wide = pp.word_bits == 64;
    const size_t words = (size_t)m * n;
    for (size_t i = 0; i < words; ++i) {  // the planes hold ceil((ct + 1) / 8) bytes of each word
        const u64 v = wide ? ((const u64 *)hint)[i] : ((const u32 *)hint)[i];
        if (v >= p) return fail(HECUDA_ERR_INVALID_ARGUMENT, "hint word >= nttFriendlyMod");
    }
    int cbd_words = 0;
    u64 cbd_mask = 0;
    if (!(pp.error_std_dev > 0 && pp.error_std_dev < 16) || !cbd_shape(pp.error_std_dev, cbd_words, cbd_mask))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "errorStdDev must be positive and below 16");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    std::string err;
    Context *ctx = Context::create(n, &p, 1, 2, err, 64);
    if (!ctx) return fail(HECUDA_ERR_UNSUPPORTED, err);
    hecuda_simple_pir_client *c = new (std::nothrow) hecuda_simple_pir_client();
    if (!c) {
        delete ctx;
        return fail(HECUDA_ERR_CUDA, "out of host memory");
    }
    cudaGetDevice(&c->device);
    c->params = pp;
    c->m = m, c->k = k, c->n = n, c->blocks = (k + n - 1) / n;
    c->entry_scalars = scalars;
    c->chunk = (scalars + pp.chunks_per_entry - 1) / pp.chunks_per_entry;
    c->p = p;
    const unsigned __int128 mu = ~(unsigned __int128)0 / p;  // floor(2^128 / p), p not a power of two
    c->mu_hi = (u64)(mu >> 64), c->mu_lo = (u64)mu;
    c->ctx = ctx;
    c->planes = spir::digits(pp.ciphertext_modulus_bits + 1);
    c->row_tiles = (m + kWarpRowTiles * spir::kTileRows - 1) / (kWarpRowTiles * spir::kTileRows) * kWarpRowTiles;
    c->col_tiles = (n + spir::kTileCols - 1) / spir::kTileCols;
    c->plane_bytes = (size_t)c->row_tiles * c->col_tiles * 512;
    c->cbd_words = cbd_words, c->cbd_mask = cbd_mask;
    cudaStream_t s = nullptr;
    void *d_hint = nullptr;
    unsigned char *d_seed = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = drbg_upload_tables(s);
    if (e == cudaSuccess) e = drbg_tables(&c->sbox, &c->te0);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_hint, c->plane_bytes * c->planes);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_a, (size_t)c->blocks * n * sizeof(u64));
    if (e == cudaSuccess) e = cudaMallocAsync(&d_hint, words * (wide ? 8 : 4), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_seed, 32, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_hint, hint, words * (wide ? 8 : 4), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seed, seed, 32, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        const long long rows_pad = c->row_tiles * spir::kTileRows;
        const unsigned grid = blocks_for(rows_pad * c->col_tiles * (spir::kTileCols / 4));
        e = wide ? launch(hint_pack_kernel<u64>, grid, kThreads, 0, s, (const u64 *)d_hint, (long long)m, (long long)n,
                          rows_pad, (long long)c->col_tiles, c->planes, c->plane_bytes, c->d_hint)
                 : launch(hint_pack_kernel<u32>, grid, kThreads, 0, s, (const u32 *)d_hint, (long long)m, (long long)n,
                          rows_pad, (long long)c->col_tiles, c->planes, c->plane_bytes, c->d_hint);
    }
    if (e == cudaSuccess) e = random_polys_one_modulus_device(d_seed, p, n, c->blocks, false, c->d_a, s);
    if (e == cudaSuccess) e = launch_ntt_forward(*ctx, ctx->map_q(1), c->d_a, c->d_a, c->blocks, s);
    for (void *q : {d_hint, (void *)d_seed})
        if (q) cudaFreeAsync(q, s);
    rc = finish_host(s, e, "simple_pir_client_create");
    if (rc) {
        hecuda_simple_pir_client_destroy(c);
        return rc;
    }
    *out = c;
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_client_destroy(hecuda_simple_pir_client *c) {
    if (!c) return HECUDA_OK;
    select_device(c->device);
    cudaDeviceSynchronize();  // no precompute in flight may still read the hint or the a-polynomials
    if (c->d_hint) cudaFree(c->d_hint);
    if (c->d_a) cudaFree(c->d_a);
    delete c->ctx;
    delete c;
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_client_precompute_device(const hecuda_simple_pir_client *c, const uint8_t *secret_seeds,
                                                   const uint8_t *error_seeds, const int64_t *indices, int64_t count,
                                                   void *queries, void *results, void *stream) {
    int32_t rc = check_call(c, count, indices, false, {secret_seeds, error_seeds, queries, results}, false);
    if (rc || count == 0) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e =
        c->params.word_bits == 64
            ? precompute_device(*c, secret_seeds, error_seeds, indices, count, (u64 *)queries, (u64 *)results, s)
            : precompute_device(*c, secret_seeds, error_seeds, indices, count, (u32 *)queries, (u32 *)results, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_client_precompute_device");
}

int32_t hecuda_simple_pir_client_precompute(const hecuda_simple_pir_client *c, const uint8_t *secret_seeds,
                                            const uint8_t *error_seeds, const int64_t *indices, int64_t count,
                                            void *queries, void *results) {
    int32_t rc = check_call(c, count, indices, false, {secret_seeds, error_seeds, queries, results}, true);
    if (rc || count == 0) return rc;
    const size_t word = c->params.word_bits / 8, cpe = c->params.chunks_per_entry;
    const size_t q_bytes = (size_t)count * cpe * c->k * word, r_bytes = (size_t)count * cpe * c->m * word;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    {
        Allocs m(s);
        unsigned char *d_ss = m.get<unsigned char>((size_t)count * 32, true), *d_es = m.get<unsigned char>((size_t)count * 32, true);
        int64_t *d_idx = indices ? m.get<int64_t>((size_t)count * sizeof(int64_t)) : nullptr;
        void *d_q = m.get<void>(q_bytes), *d_r = m.get<void>(r_bytes, true);
        if (e == cudaSuccess) e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_ss, secret_seeds, (size_t)count * 32, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_es, error_seeds, (size_t)count * 32, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && indices) e = cudaMemcpyAsync(d_idx, indices, (size_t)count * 8, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess)
            e = word == 8 ? precompute_device(*c, d_ss, d_es, d_idx, count, (u64 *)d_q, (u64 *)d_r, s)
                          : precompute_device(*c, d_ss, d_es, d_idx, count, (u32 *)d_q, (u32 *)d_r, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(queries, d_q, q_bytes, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(results, d_r, r_bytes, cudaMemcpyDeviceToHost, s);
    }
    return finish_host(s, e, "simple_pir_client_precompute");
}

int32_t hecuda_simple_pir_client_decrypt_device(const hecuda_simple_pir_client *c, const void *responses, const void *results,
                                                const int64_t *indices, int64_t count, uint8_t *entries, void *stream) {
    int32_t rc = check_call(c, count, indices, true, {responses, results, entries}, false);
    if (rc || count == 0) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = c->params.word_bits == 64
                              ? decrypt_device(*c, (const u64 *)responses, (const u64 *)results, indices, count, entries, s)
                              : decrypt_device(*c, (const u32 *)responses, (const u32 *)results, indices, count, entries, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_client_decrypt_device");
}

int32_t hecuda_simple_pir_client_decrypt(const hecuda_simple_pir_client *c, const void *responses, const void *results,
                                         const int64_t *indices, int64_t count, uint8_t *entries) {
    int32_t rc = check_call(c, count, indices, true, {responses, results, entries}, true);
    if (rc || count == 0) return rc;
    const size_t word = c->params.word_bits / 8;
    const size_t bytes = (size_t)count * c->params.chunks_per_entry * c->m * word, out = (size_t)count * c->params.entry_size;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    {
        Allocs m(s);
        void *d_resp = m.get<void>(bytes), *d_res = m.get<void>(bytes, true);
        int64_t *d_idx = m.get<int64_t>((size_t)count * sizeof(int64_t));
        unsigned char *d_out = m.get<unsigned char>(out, true);
        if (e == cudaSuccess) e = m.e;
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_resp, responses, bytes, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_res, results, bytes, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_idx, indices, (size_t)count * 8, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess)
            e = word == 8 ? decrypt_device(*c, (const u64 *)d_resp, (const u64 *)d_res, d_idx, count, d_out, s)
                          : decrypt_device(*c, (const u32 *)d_resp, (const u32 *)d_res, d_idx, count, d_out, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(entries, d_out, out, cudaMemcpyDeviceToHost, s);
    }
    return finish_host(s, e, "simple_pir_client_decrypt");
}

}  // extern "C"
