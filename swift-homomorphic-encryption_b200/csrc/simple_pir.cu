// simple_pir.cu -- SimplePIR's server on the device: the processed database as resident u8 digit planes, its hint
// DB' . A mod p through the negacyclic structure of A, and batched responses (DB' . request^T) mod 2^ct on the integer
// tensor cores (mma.sync m16n8k32 u8 x u8 -> s32).  The arithmetic and index maps are in simple_pir.cuh.
//
//   SimplePirServer.process               SimplePir/SimplePir+Database.swift:252-290
//   SimplePirContext.generateAPolynomials / materializeAMatrix   :177-206
//   SimplePirServer(processedDatabase:hint:params:), computeResponse   SimplePir+Server.swift:24-38
#include <algorithm>
#include <vector>

#include "capi_internal.hpp"
#include "hostmath.hpp"
#include "ntt_fast.cuh"
#include "simple_pir.cuh"

using namespace hecuda;
using namespace hecuda::api;

struct hecuda_simple_pir_database {
    int device = 0;
    hecuda_simple_pir_params params{};
    int64_t m = 0, k = 0;             // DB' is m x k (columnSize x databaseColumns)
    int64_t row_tiles = 0, col_tiles = 0;  // 16-row / 32-column tiles of a plane (rows padded to kWarpRowTiles tiles)
    int planes = 0;                   // ceil(pt / 8)
    size_t plane_bytes = 0;
    unsigned char *d_planes = nullptr;  // planes x plane_bytes (simple_pir.cuh, a_offset)
};

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = 4;            // response kernel: warps per CTA, stacked over rows
constexpr int kWarpRowTiles = 2;     // 16-row tiles per warp
constexpr int kCtaQueryTiles = 2;    // 8-query tiles per CTA (every warp of a CTA reads the same request tiles)
constexpr int kMinSplitTiles = 64;   // smallest K range (in 32-column tiles) one CTA of a split-K launch takes
constexpr int64_t kHintSlabWords = 32ll << 20;  // hint: <= 256 MB of forward-NTT rows per slab

struct Geometry {
    int64_t m, k, row_tiles, col_tiles;
    int planes;
    size_t plane_bytes;
};

// ---- digit planes
__device__ __forceinline__ void store_digits(unsigned char *planes, size_t plane_bytes, int count, long long at,
                                             const u64 v[4]) {
    for (int i = 0; i < count; ++i) {
        unsigned w = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) w |= spir::db_digit(v[b], i) << (8 * b);
        *reinterpret_cast<unsigned *>(planes + i * plane_bytes + at) = w;
    }
}

__device__ __forceinline__ u64 plane_value(const unsigned char *planes, size_t plane_bytes, int count, long long r,
                                           long long c, long long col_tiles) {
    const long long at = spir::a_offset(r, c, col_tiles);
    u64 v = 0;
    for (int i = 0; i < count; ++i) v |= (u64)planes[i * plane_bytes + at] << (8 * i);
    return v;
}

// process's packing and transpose: thread (r, four columns) of the padded plane; adjacent threads take adjacent rows,
// which are adjacent coefficients of one entry
__global__ void __launch_bounds__(kThreads) pack_entries_kernel(const procdb::PirShape s, const Geometry g, long long padded_entry,
                                                                long long entry_scalars, unsigned char *__restrict__ planes) {
    const long long rows = g.row_tiles * spir::kTileRows;
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows * g.col_tiles * (spir::kTileCols / 4)) return;
    const long long r = t % rows, c0 = t / rows * 4;
    u64 v[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        long long e = -1, k = 0;
        if (r < g.m && c0 + b < g.k) spir::db_source(r, c0 + b, g.m, padded_entry, entry_scalars, s.entry_count, e, k);
        v[b] = e < 0 ? 0 : procdb::pir_coefficient(s, procdb::PirPiece{e, 0, s.entry_size}, k);
    }
    store_digits(planes, g.plane_bytes, g.planes, spir::a_offset(r, c0, g.col_tiles), v);
}

// SimplePirServer(processedDatabase:): the m x k matrix (values < 2^pt, checked on the host) into the planes
template <typename W>
__global__ void __launch_bounds__(kThreads) pack_matrix_kernel(const W *__restrict__ matrix, const Geometry g,
                                                               unsigned char *__restrict__ planes) {
    const long long rows = g.row_tiles * spir::kTileRows, quads = g.col_tiles * (spir::kTileCols / 4);
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows * quads) return;
    const long long c0 = t % quads * 4, r = t / quads;
    u64 v[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) v[b] = r < g.m && c0 + b < g.k ? (u64)matrix[r * g.k + c0 + b] : 0;
    store_digits(planes, g.plane_bytes, g.planes, spir::a_offset(r, c0, g.col_tiles), v);
}

template <typename W>
__global__ void __launch_bounds__(kThreads) export_kernel(const unsigned char *__restrict__ planes, const Geometry g,
                                                          W *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= g.m * g.k) return;
    out[t] = (W)plane_value(planes, g.plane_bytes, g.planes, t / g.k, t % g.k, g.col_tiles);
}

// ---- hint: rows r0 .. r0 + rows of DB' as rows x ceil(k / n) blocks of n columns, zero past k
__global__ void __launch_bounds__(kThreads) hint_fill_kernel(const unsigned char *__restrict__ planes, const Geometry g,
                                                             long long r0, long long rows, long long padded_cols,
                                                             u64 *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= rows * padded_cols) return;
    const long long rl = t / padded_cols, c = t - rl * padded_cols;
    out[t] = c < g.k ? plane_value(planes, g.plane_bytes, g.planes, r0 + rl, c, g.col_tiles) : 0;
}

// ---- response
// requests q x k words -> digit planes (simple_pir.cuh, b_offset), zero past q and k; thread (query, four columns)
template <typename W>
__global__ void __launch_bounds__(kThreads) split_requests_kernel(const W *__restrict__ req, long long q, long long k,
                                                                  long long q_pad, long long col_tiles, int ct, int digits,
                                                                  unsigned char *__restrict__ out, long long plane_bytes) {
    const long long quads = col_tiles * (spir::kTileCols / 4);
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= q_pad * quads) return;
    const long long c0 = t % quads * 4, row = t / quads;
    u64 w[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) w[b] = row < q && c0 + b < k ? (u64)req[row * k + c0 + b] : 0;
    const long long at = spir::b_offset(row, c0, col_tiles);
    for (int j = 0; j < digits; ++j) {
        unsigned d = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) d |= spir::query_digit(w[b], ct, j) << (8 * b);
        *reinterpret_cast<unsigned *>(out + j * plane_bytes + at) = d;
    }
}

__device__ __forceinline__ void mma_u8(int (&c)[4], const uint4 &a, const uint2 &b) {
    asm volatile(
        "mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b.x), "r"(b.y));
}

struct ResponseArgs {
    const unsigned char *planes;
    size_t plane_bytes;
    int planes_count;
    const unsigned char *digits;  // request digit planes
    long long digit_plane_bytes;
    long long col_tiles, m, q;
    long long split_tiles;  // 32-column tiles per blockIdx.z
    int ct;
};

// Warp w of a CTA owns row tiles (blockIdx.x * kWarps + w) * 2 + {0, 1} and query tiles query_tile0 + blockIdx.y * 2 +
// {0, 1}, over the K range of blockIdx.z.  For every slice of <= kSliceTiles tiles and every plane i, the s32 sums of
// each live (i, j) pair are accumulated by the MMA and then widened into the 64-bit sums; the K ranges' sums meet in
// acc (mod 2^64, so the order of the atomic adds does not matter).
template <int D>
__global__ void __launch_bounds__(kWarps * 32) response_kernel(const ResponseArgs a, long long query_tile0, u64 *__restrict__ acc) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long rt0 = ((long long)blockIdx.x * kWarps + warp) * kWarpRowTiles;
    if (rt0 * spir::kTileRows >= a.m) return;  // padding rows only; the kernel has no block-wide barrier
    const long long qt0 = query_tile0 + (long long)blockIdx.y * kCtaQueryTiles;
    const long long kt_begin = (long long)blockIdx.z * a.split_tiles;
    const long long kt_end = min(a.col_tiles, kt_begin + a.split_tiles);
    u64 wide[kWarpRowTiles][kCtaQueryTiles][4];
#pragma unroll
    for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
        for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) wide[mt][nt][e] = 0;
    for (long long s0 = kt_begin; s0 < kt_end; s0 += spir::kSliceTiles) {
        const long long s1 = min(kt_end, s0 + spir::kSliceTiles);
        for (int i = 0; i < a.planes_count; ++i) {
            int sum[kWarpRowTiles][D][kCtaQueryTiles][4];
#pragma unroll
            for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
                for (int j = 0; j < D; ++j)
#pragma unroll
                    for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
                        for (int e = 0; e < 4; ++e) sum[mt][j][nt][e] = 0;
            const uint4 *pa = reinterpret_cast<const uint4 *>(a.planes + i * a.plane_bytes) + rt0 * a.col_tiles * 32 + lane;
            for (long long kt = s0; kt < s1; ++kt) {
                uint4 fa[kWarpRowTiles];
#pragma unroll
                for (int mt = 0; mt < kWarpRowTiles; ++mt) fa[mt] = __ldcs(pa + (mt * a.col_tiles + kt) * 32);
#pragma unroll
                for (int j = 0; j < D; ++j) {
                    if (!spir::pair_live(i, j, a.ct)) continue;
                    const uint2 *pb = reinterpret_cast<const uint2 *>(a.digits + j * a.digit_plane_bytes) + lane;
#pragma unroll
                    for (int nt = 0; nt < kCtaQueryTiles; ++nt) {
                        const uint2 fb = __ldg(pb + ((qt0 + nt) * a.col_tiles + kt) * 32);
#pragma unroll
                        for (int mt = 0; mt < kWarpRowTiles; ++mt) mma_u8(sum[mt][j][nt], fa[mt], fb);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < D; ++j) {
                if (!spir::pair_live(i, j, a.ct)) continue;
#pragma unroll
                for (int mt = 0; mt < kWarpRowTiles; ++mt)
#pragma unroll
                    for (int nt = 0; nt < kCtaQueryTiles; ++nt)
#pragma unroll
                        for (int e = 0; e < 4; ++e) wide[mt][nt][e] = spir::widen(wide[mt][nt][e], (u32)sum[mt][j][nt][e], i, j);
            }
        }
    }
    // C fragment: e = 0, 1 at (row g, queries 2t, 2t + 1), e = 2, 3 at row g + 8
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
                    atomicAdd(reinterpret_cast<unsigned long long *>(acc + query * a.m + row),
                              (unsigned long long)wide[mt][nt][e]);
            }
}

// responses[q][r] = acc[q][r] mod 2^ct in the reference's scalar width (query q = request * chunksPerEntry + chunk)
template <typename W>
__global__ void __launch_bounds__(kThreads) finish_kernel(const u64 *__restrict__ acc, long long words, int ct, W *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t < words) out[t] = (W)spir::finish(acc[t], ct);
}

unsigned blocks_for(long long threads) { return (unsigned)((threads + kThreads - 1) / kThreads); }

// ---- parameters: SimplePirEncryptionParams / SimplePirParameters (SimplePir.swift:47-79, 95-160)
struct Derived {
    int64_t entry_scalars, padded_entry, m, k;
    u64 p;
    Geometry g;
};

int64_t coeff_count(int64_t bytes, int bits) { return (bytes * 8 + bits - 1) / bits; }  // bytesToCoefficientsCoeffCount

int32_t derive(const hecuda_simple_pir_params *pp, Derived &d) {
    if (!pp) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const hecuda_simple_pir_params &p = *pp;
    const int64_t n = p.lattice_dimension;
    if (n < 2 || (n & (n - 1)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidEncryptionParameters: SimplePir latticeDimension is not a power of 2");
    if (p.plaintext_modulus_bits < 1 || p.ciphertext_modulus_bits <= p.plaintext_modulus_bits)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidEncryptionParameters: SimplePir ciphertextModulusBits must be > plaintextModulusBits");
    if (p.word_bits != 32 && p.word_bits != 64) return fail(HECUDA_ERR_INVALID_ARGUMENT, "word_bits must be 32 or 64");
    if (p.entry_size < 1 || p.entries_per_column < 1 || p.chunks_per_entry < 1 || p.database_columns < 1)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePirParameters: sizes must be positive");
    if (p.entries_per_column != 1 && p.chunks_per_entry != 1)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePirParameters: entriesPerColumn == 1 || chunksPerEntry == 1");
    if (n > (1 << fast::kSplitLogN))
        return fail(HECUDA_ERR_UNSUPPORTED, "unsupportedHeOperation: latticeDimension above the NTT kernels' largest degree");
    // nttFriendlyMod: the smallest (ct + 1)-bit prime = 1 mod 2N (SimplePirContext.swift:78-81); generatePrimes fails
    // above the scalar width, and the device context keeps moduli below 2^62
    const int ct = p.ciphertext_modulus_bits;
    if (ct + 1 > p.word_bits) return fail(HECUDA_ERR_UNSUPPORTED, "ciphertextModulusBits + 1 exceeds the scalar width");
    if (ct + 1 > 62) return fail(HECUDA_ERR_UNSUPPORTED, "nttFriendlyMod must be below 2^62");
    const std::vector<u64> primes = host::smallest_ntt_primes(ct + 1, 1, (u64)n);
    if (primes.empty()) return fail(HECUDA_ERR_UNSUPPORTED, "notEnoughPrimes: no NTT-friendly prime of ciphertextModulusBits + 1 bits");
    d.p = primes[0];
    const int pt = p.plaintext_modulus_bits;
    if (p.entry_size > (1ll << 40) || p.database_columns > (1ll << 40)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePirParameters: size out of range");
    d.entry_scalars = coeff_count(p.entry_size, pt);
    const int64_t cpe = p.chunks_per_entry, epc = p.entries_per_column;
    d.padded_entry = cpe == 1 ? d.entry_scalars : (d.entry_scalars + cpe - 1) / cpe * cpe;
    d.m = cpe == 1 ? epc * d.entry_scalars : (d.entry_scalars + cpe - 1) / cpe;  // columnSize
    d.k = p.database_columns;
    if (d.m > (1ll << 31) || (double)d.m * (double)d.k > 4e12) return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePirParameters: database too large");
    Geometry &g = d.g;
    g.m = d.m;
    g.k = d.k;
    g.row_tiles = (d.m + kWarpRowTiles * spir::kTileRows - 1) / (kWarpRowTiles * spir::kTileRows) * kWarpRowTiles;
    g.col_tiles = (d.k + spir::kTileCols - 1) / spir::kTileCols;
    g.planes = spir::digits(pt);
    g.plane_bytes = (size_t)g.row_tiles * g.col_tiles * 512;
    return HECUDA_OK;
}

int32_t select_device(int device) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device available");
    if (dev != device) CK(cudaSetDevice(device));
    return HECUDA_OK;
}

hecuda_simple_pir_database *new_database(const hecuda_simple_pir_params &p, const Derived &d) {
    hecuda_simple_pir_database *db = new (std::nothrow) hecuda_simple_pir_database();
    if (!db) return nullptr;
    cudaGetDevice(&db->device);
    db->params = p;
    db->m = d.m;
    db->k = d.k;
    db->row_tiles = d.g.row_tiles;
    db->col_tiles = d.g.col_tiles;
    db->planes = d.g.planes;
    db->plane_bytes = d.g.plane_bytes;
    return db;
}

Geometry geometry(const hecuda_simple_pir_database &db) {
    return Geometry{db.m, db.k, db.row_tiles, db.col_tiles, db.planes, db.plane_bytes};
}

// hint = DB' . A mod p (M x N) = coeffs(sum_j sigma(a_j) . d_{r,j}) per row (DESIGN.md): one forward NTT per (row, block),
// the lazy Eval-domain inner product against NTT(sigma(a_j)), one inverse NTT per row; d_hint: M x N u64
cudaError_t compute_hint(const Context &ctx, const hecuda_simple_pir_database &db, const unsigned char *d_seed, u64 *d_hint,
                         cudaStream_t s) {
    const int64_t n = ctx.n, blocks = (db.k + n - 1) / n;  // aPolyCount
    const NttRowMap map = ctx.map_q(1);
    const Geometry g = geometry(db);
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(db.m, kHintSlabWords / (blocks * n)));
    u64 *d_a = nullptr, *d_rows = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_a, (size_t)blocks * n * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_rows, (size_t)slab * blocks * n * sizeof(u64), s);
    if (e == cudaSuccess) e = random_sigma_polys_device(d_seed, ctx.q[0], n, blocks, d_a, s);
    if (e == cudaSuccess) e = launch_ntt_forward(ctx, map, d_a, d_a, blocks, s);
    for (int64_t r0 = 0; e == cudaSuccess && r0 < db.m; r0 += slab) {
        const int64_t rows = std::min(slab, db.m - r0);
        u64 *out = d_hint + r0 * n;
        e = launch(hint_fill_kernel, blocks_for(rows * blocks * n), kThreads, 0, s, (const unsigned char *)db.d_planes, g,
                   (long long)r0, (long long)rows, (long long)(blocks * n), d_rows);
        if (e == cudaSuccess) e = launch_ntt_forward(ctx, map, d_rows, d_rows, rows * blocks, s);
        if (e == cudaSuccess) e = launch_inner_product_plain(ctx, d_a, 1, 1, blocks, d_rows, nullptr, out, rows, s);
        if (e == cudaSuccess) e = launch_ntt_inverse(ctx, map, out, out, rows, kScalePlain, s);
    }
    if (d_a) cudaFreeAsync(d_a, s);
    if (d_rows) cudaFreeAsync(d_rows, s);
    return e;
}

template <int D>
cudaError_t launch_response(const ResponseArgs &a, int64_t query_tiles, int sm_count, u64 *acc, cudaStream_t s) {
    const unsigned gx = (unsigned)((a.col_tiles ? (a.m + kWarps * kWarpRowTiles * spir::kTileRows - 1) /
                                                      (kWarps * kWarpRowTiles * spir::kTileRows)
                                                : 0));
    const int64_t pairs = query_tiles / kCtaQueryTiles;
    // split K until the grid covers the SMs about four times over, with at least kMinSplitTiles tiles per CTA
    const int64_t ctas = (int64_t)gx * std::min<int64_t>(pairs, kMaxGridYZ);
    int64_t splits = std::max<int64_t>(1, (4ll * sm_count + ctas - 1) / ctas);
    splits = std::min<int64_t>({splits, std::max<int64_t>(1, a.col_tiles / kMinSplitTiles), kMaxGridYZ});
    ResponseArgs args = a;
    args.split_tiles = (a.col_tiles + splits - 1) / splits;
    splits = (a.col_tiles + args.split_tiles - 1) / args.split_tiles;
    return for_each_part(pairs, [&](int64_t first, int64_t part) {
        return launch(response_kernel<D>, dim3(gx, (unsigned)part, (unsigned)splits), kWarps * 32, 0, s, args,
                      (long long)(first * kCtaQueryTiles), acc);
    });
}

// computeResponse for `count` requests already on the device, enqueued on s
template <typename W>
cudaError_t response_device(const hecuda_simple_pir_database &db, const W *d_req, int64_t count, W *d_out, cudaStream_t s) {
    const int ct = db.params.ciphertext_modulus_bits, digits = spir::digits(ct);
    const int64_t q = count * db.params.chunks_per_entry;
    const int64_t q_tile_span = (int64_t)spir::kTileQueries * kCtaQueryTiles;
    const int64_t q_pad = (q + q_tile_span - 1) / q_tile_span * q_tile_span;
    const long long digit_plane = (long long)q_pad * db.col_tiles * spir::kTileCols;
    int dev = 0, sms = 1;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    unsigned char *d_digits = nullptr;
    u64 *d_acc = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_digits, (size_t)digit_plane * digits, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_acc, (size_t)q * db.m * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_acc, 0, (size_t)q * db.m * sizeof(u64), s);
    if (e == cudaSuccess)
        e = launch(split_requests_kernel<W>, blocks_for(q_pad * db.col_tiles * (spir::kTileCols / 4)), kThreads, 0, s, d_req,
                   (long long)q, (long long)db.k, (long long)q_pad, (long long)db.col_tiles, ct, digits, d_digits, digit_plane);
    if (e == cudaSuccess) {
        const ResponseArgs a{db.d_planes, db.plane_bytes, db.planes, d_digits, digit_plane, (long long)db.col_tiles,
                             (long long)db.m, (long long)q, 0, ct};
        const int64_t tiles = q_pad / spir::kTileQueries;
        switch (digits) {
            case 1: e = launch_response<1>(a, tiles, sms, d_acc, s); break;
            case 2: e = launch_response<2>(a, tiles, sms, d_acc, s); break;
            case 3: e = launch_response<3>(a, tiles, sms, d_acc, s); break;
            case 4: e = launch_response<4>(a, tiles, sms, d_acc, s); break;
            case 5: e = launch_response<5>(a, tiles, sms, d_acc, s); break;
            case 6: e = launch_response<6>(a, tiles, sms, d_acc, s); break;
            case 7: e = launch_response<7>(a, tiles, sms, d_acc, s); break;
            default: e = launch_response<8>(a, tiles, sms, d_acc, s); break;
        }
    }
    if (e == cudaSuccess) e = launch(finish_kernel<W>, blocks_for(q * db.m), kThreads, 0, s, (const u64 *)d_acc, (long long)(q * db.m), ct, d_out);
    if (d_digits) cudaFreeAsync(d_digits, s);
    if (d_acc) cudaFreeAsync(d_acc, s);
    return e;
}

int32_t check_response(const hecuda_simple_pir_database *db, const void *req, int64_t count, const void *out) {
    if (!db) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null database");
    if (count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative request count");
    if (count && (!req || !out)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    if (count > (1ll << 40) / std::max<int64_t>(1, db->params.chunks_per_entry * std::max(db->k, db->m)))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "too many requests for one call");
    return select_device(db->device);
}

}  // namespace

extern "C" {

int32_t hecuda_simple_pir_process(const uint8_t *entries, int64_t entry_count, const hecuda_simple_pir_params *params,
                                  const uint8_t *seed, void *hint, hecuda_simple_pir_database **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    Derived d;
    int32_t rc = derive(params, d);
    if (rc) return rc;
    if (!entries || !seed || !hint) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (entry_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "empty database");
    if ((double)entry_count * (double)d.padded_entry > (double)d.m * (double)d.k ||
        entry_count * d.padded_entry > d.m * d.k)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "SimplePirParameters: the entries do not fit databaseColumns x columnSize");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    // the single-modulus context of the hint (extraContext, SimplePirContext.swift:82); t only has to be below p
    std::string err;
    Context *ctx = Context::create(params->lattice_dimension, &d.p, 1, 2, err, 64);
    if (!ctx) return fail(HECUDA_ERR_UNSUPPORTED, err);
    hecuda_simple_pir_database *db = new_database(*params, d);
    if (!db) {
        delete ctx;
        return fail(HECUDA_ERR_CUDA, "out of host memory");
    }
    const size_t entry_bytes = (size_t)entry_count * params->entry_size;
    const int64_t n = params->lattice_dimension;
    const size_t hint_words = (size_t)d.m * n;
    cudaStream_t s = nullptr;
    unsigned char *d_entries = nullptr, *d_seed = nullptr;
    u64 *d_hint = nullptr;
    u32 *d_hint32 = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&db->d_planes, db->plane_bytes * db->planes);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_entries, entry_bytes, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_seed, 32, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_hint, hint_words * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_entries, entries, entry_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seed, seed, 32, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        procdb::PirShape ps{};
        ps.entries = d_entries;
        ps.entry_count = entry_count;
        ps.entry_size = params->entry_size;
        ps.encoded = params->entry_size;
        ps.bits = params->plaintext_modulus_bits;
        const Geometry g = d.g;
        e = launch(pack_entries_kernel, blocks_for(g.row_tiles * spir::kTileRows * g.col_tiles * (spir::kTileCols / 4)),
                   kThreads, 0, s, ps, g, (long long)d.padded_entry, (long long)d.entry_scalars, db->d_planes);
    }
    if (d_entries) cudaFreeAsync(d_entries, s);
    if (e == cudaSuccess) e = compute_hint(*ctx, *db, d_seed, d_hint, s);
    if (e == cudaSuccess) {
        if (params->word_bits == 64) {
            e = cudaMemcpyAsync(hint, d_hint, hint_words * sizeof(u64), cudaMemcpyDeviceToHost, s);
        } else {
            e = cudaMallocAsync((void **)&d_hint32, hint_words * sizeof(u32), s);
            if (e == cudaSuccess) e = launch_narrow(d_hint, d_hint32, (int64_t)hint_words, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(hint, d_hint32, hint_words * sizeof(u32), cudaMemcpyDeviceToHost, s);
        }
    }
    for (void *p : {(void *)d_seed, (void *)d_hint, (void *)d_hint32})
        if (p) cudaFreeAsync(p, s);
    if (s) {
        const cudaError_t e2 = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(s);
    }
    delete ctx;
    if (e != cudaSuccess) {
        hecuda_simple_pir_database_destroy(db);
        return cuda_fail(e, "simple_pir_process");
    }
    *out = db;
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_database_create(const void *processed, const hecuda_simple_pir_params *params,
                                          hecuda_simple_pir_database **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    Derived d;
    int32_t rc = derive(params, d);
    if (rc) return rc;
    if (!processed) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const size_t words = (size_t)d.m * d.k;
    const int pt = params->plaintext_modulus_bits;
    const bool wide = params->word_bits == 64;
    for (size_t i = 0; i < words; ++i) {  // the digit planes hold pt bits
        const u64 v = wide ? ((const u64 *)processed)[i] : ((const u32 *)processed)[i];
        if (v >> pt) return fail(HECUDA_ERR_INVALID_ARGUMENT, "processed database value >= 2^plaintextModulusBits");
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    hecuda_simple_pir_database *db = new_database(*params, d);
    if (!db) return fail(HECUDA_ERR_CUDA, "out of host memory");
    const size_t bytes = words * (wide ? 8 : 4);
    void *d_matrix = nullptr;
    cudaError_t e = cudaMalloc(&db->d_planes, db->plane_bytes * db->planes);
    if (e == cudaSuccess) e = cudaMalloc(&d_matrix, bytes);
    if (e == cudaSuccess) e = upload(d_matrix, processed, bytes);
    const Geometry g = d.g;
    const unsigned grid = blocks_for(g.row_tiles * spir::kTileRows * g.col_tiles * (spir::kTileCols / 4));
    if (e == cudaSuccess)
        e = wide ? launch(pack_matrix_kernel<u64>, grid, kThreads, 0, cudaStreamLegacy, (const u64 *)d_matrix, g, db->d_planes)
                 : launch(pack_matrix_kernel<u32>, grid, kThreads, 0, cudaStreamLegacy, (const u32 *)d_matrix, g, db->d_planes);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    if (d_matrix) cudaFree(d_matrix);
    if (e != cudaSuccess) {
        hecuda_simple_pir_database_destroy(db);
        return cuda_fail(e, "simple_pir_database_create");
    }
    *out = db;
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_database_export(const hecuda_simple_pir_database *db, void *processed) {
    if (!db || !processed) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = select_device(db->device);
    if (rc) return rc;
    const bool wide = db->params.word_bits == 64;
    const size_t words = (size_t)db->m * db->k, bytes = words * (wide ? 8 : 4);
    const Geometry g = geometry(*db);
    void *d_matrix = nullptr;
    cudaError_t e = cudaMalloc(&d_matrix, bytes);
    if (e == cudaSuccess)
        e = wide ? launch(export_kernel<u64>, blocks_for((long long)words), kThreads, 0, cudaStreamLegacy,
                          (const unsigned char *)db->d_planes, g, (u64 *)d_matrix)
                 : launch(export_kernel<u32>, blocks_for((long long)words), kThreads, 0, cudaStreamLegacy,
                          (const unsigned char *)db->d_planes, g, (u32 *)d_matrix);
    if (e == cudaSuccess) e = cudaMemcpy(processed, d_matrix, bytes, cudaMemcpyDeviceToHost);
    if (d_matrix) cudaFree(d_matrix);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_database_export");
}

int32_t hecuda_simple_pir_database_destroy(hecuda_simple_pir_database *db) {
    if (!db) return HECUDA_OK;
    if (db->d_planes) {
        select_device(db->device);
        cudaDeviceSynchronize();  // no response in flight may still read the planes
        cudaFree(db->d_planes);
    }
    delete db;
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_compute_response_device(const hecuda_simple_pir_database *db, const void *requests, int64_t count,
                                                  void *responses, void *stream) {
    int32_t rc = check_response(db, requests, count, responses);
    if (rc || count == 0) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = db->params.word_bits == 64
                              ? response_device(*db, (const u64 *)requests, count, (u64 *)responses, s)
                              : response_device(*db, (const u32 *)requests, count, (u32 *)responses, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_compute_response_device");
}

int32_t hecuda_simple_pir_compute_response(const hecuda_simple_pir_database *db, const void *requests, int64_t count,
                                           void *responses) {
    int32_t rc = check_response(db, requests, count, responses);
    if (rc || count == 0) return rc;
    const size_t word = db->params.word_bits / 8, cpe = db->params.chunks_per_entry;
    const size_t in_bytes = (size_t)count * cpe * db->k * word, out_bytes = (size_t)count * cpe * db->m * word;
    cudaStream_t s = nullptr;
    void *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_in, in_bytes, s);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_out, out_bytes, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, requests, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess)
        e = word == 8 ? response_device(*db, (const u64 *)d_in, count, (u64 *)d_out, s)
                      : response_device(*db, (const u32 *)d_in, count, (u32 *)d_out, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(responses, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
    for (void *p : {d_in, d_out})
        if (p) cudaFreeAsync(p, s);
    if (s) {
        const cudaError_t e2 = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(s);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_compute_response");
}

}  // extern "C"
