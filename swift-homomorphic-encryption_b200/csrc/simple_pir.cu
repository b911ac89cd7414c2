// simple_pir.cu -- SimplePIR's server on the device: the processed database as resident u8 digit planes, its hint
// DB' . A mod p through the negacyclic structure of A, and batched responses (DB' . request^T) mod 2^ct on the integer
// tensor cores (mma.sync m16n8k32 u8 x u8 -> s32).  The arithmetic and index maps are in simple_pir.cuh.
//
//   SimplePirServer.process               SimplePir/SimplePir+Database.swift:252-290
//   SimplePirContext.generateAPolynomials / materializeAMatrix   :177-206
//   SimplePirServer(processedDatabase:hint:params:), computeResponse   SimplePir+Server.swift:24-38
//   DatabaseMap.shardDatabase + per-shard process   SimplePir/DatabaseMap.swift:82-110, SimplePIRProcessDatabase/main.swift:158-253
//   every shard's responses for SimplePirClientForAllShards   SimplePir/SimplePir+Shards.swift:47-173
//   SimplePIRRequest in, SimplePIRResponse out   PirConversion.swift:380-401, SimplePir+Server.swift:31-38
#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

#include "capi_internal.hpp"
#include "hostmath.hpp"
#include "ntt_fast.cuh"
#include "simple_pir.cuh"
#include "simple_pir_proto.hpp"

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

// pack_entries_kernel for one shard: its row e is the chunk row_source[e] = {entry, chunk} of the raw entries
__global__ void __launch_bounds__(kThreads) pack_shard_kernel(const procdb::PirShape s, const Geometry g, long long padded_entry,
                                                              long long entry_scalars, long long rows,
                                                              const long long *__restrict__ row_source, long long chunk_size,
                                                              unsigned char *__restrict__ planes) {
    const long long padded_rows = g.row_tiles * spir::kTileRows;
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= padded_rows * g.col_tiles * (spir::kTileCols / 4)) return;
    const long long r = t % padded_rows, c0 = t / padded_rows * 4;
    u64 v[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        long long e = -1, k = 0;
        if (r < g.m && c0 + b < g.k) spir::db_source(r, c0 + b, g.m, padded_entry, entry_scalars, rows, e, k);
        v[b] = e < 0 ? 0
                     : procdb::pir_coefficient(s, spir::shard_piece(s, row_source[2 * e], row_source[2 * e + 1], chunk_size), k);
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

using spir::mma_u8;

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

static_assert(spir::kCtaRows == kWarps * kWarpRowTiles * spir::kTileRows, "simple_pir.cuh's CTA rows");
static_assert(spir::kCtaQueries == kCtaQueryTiles * spir::kTileQueries, "simple_pir.cuh's CTA queries");

// One warp's share of a response CTA: row tiles rt0 + {0, 1} against query tiles qt0 + {0, 1} over the K tiles
// [kt_begin, kt_end).  For every slice of <= kSliceTiles tiles and every plane i, the s32 sums of each live (i, j) pair
// are accumulated by the MMA and then widened into the 64-bit sums, which are atomically added at at(query, row) for
// every row < a.m and query < a.q.
template <int D, typename At>
__device__ __forceinline__ void response_warp(const ResponseArgs &a, long long rt0, long long qt0, long long kt_begin,
                                              long long kt_end, int lane, At at) {
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
                    atomicAdd(reinterpret_cast<unsigned long long *>(at(query, row)), (unsigned long long)wide[mt][nt][e]);
            }
}

// Warp w of a CTA owns row tiles (blockIdx.x * kWarps + w) * 2 + {0, 1} and query tiles query_tile0 + blockIdx.y * 2 +
// {0, 1}, over the K range of blockIdx.z; the K ranges' sums meet in acc (mod 2^64, so the order of the atomic adds
// does not matter).
template <int D>
__global__ void __launch_bounds__(kWarps * 32) response_kernel(const ResponseArgs a, long long query_tile0, u64 *__restrict__ acc) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long rt0 = ((long long)blockIdx.x * kWarps + warp) * kWarpRowTiles;
    if (rt0 * spir::kTileRows >= a.m) return;  // padding rows only; the kernel has no block-wide barrier
    const long long qt0 = query_tile0 + (long long)blockIdx.y * kCtaQueryTiles;
    const long long kt_begin = (long long)blockIdx.z * a.split_tiles;
    const long long kt_end = min(a.col_tiles, kt_begin + a.split_tiles);
    response_warp<D>(a, rt0, qt0, kt_begin, kt_end, lane,
                     [&](long long query, long long row) { return acc + query * a.m + row; });
}

// ---- grouped responses over shards (simple_pir.cuh, "grouped responses").  Requests and responses are client-major:
// client c's block holds, for each shard s in order, requests_per_shard x chunksPerEntry_s rows of K_s request words
// (M_s response words).  Query q of shard s is row q % qpc of client q / qpc's part of shard s.  The accumulators use
// the responses' layout, so one finish_kernel serves every shard.
constexpr int kMaxShards = 32;  // shards per launch: their descriptors travel in the kernel parameters

struct ShardDesc {
    const unsigned char *planes;
    unsigned char *digits;  // the shard's request digit planes
    size_t plane_bytes;
    long long m, k, q;       // DB' rows and columns, queries (count x qpc)
    long long split_tiles;   // 32-column tiles per K range
    long long qpc;           // queries per client: requests_per_shard x chunksPerEntry
    long long in_off, out_off;  // the shard's first word in a client's request / response block
};

struct ShardGroup {
    int count, planes, ct;
    long long in_block, out_block;  // words per client, over every shard of the call
    long long split_threads;        // split_shards_kernel threads of the group
    long long item_begin[kMaxShards], split_begin[kMaxShards];
    ShardDesc shard[kMaxShards];
};
static_assert(sizeof(ShardGroup) < 4096, "the grouped kernels' parameters must stay under 4 KB");

__device__ __forceinline__ long long col_tiles_of(long long k) { return (k + spir::kTileCols - 1) / spir::kTileCols; }
__device__ __forceinline__ long long digit_plane_of(const ShardDesc &d) {
    return (d.q + spir::kCtaQueries - 1) / spir::kCtaQueries * spir::kCtaQueries * col_tiles_of(d.k) * spir::kTileCols;
}

// split_requests_kernel for every shard of the group: thread (shard, query, four columns)
template <typename W>
__global__ void __launch_bounds__(kThreads) split_shards_kernel(const W *__restrict__ req, const ShardGroup g) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= g.split_threads) return;
    const int s = spir::item_shard(g.split_begin, g.count, t);
    const ShardDesc &d = g.shard[s];
    const long long col_tiles = col_tiles_of(d.k), quads = col_tiles * (spir::kTileCols / 4);
    const long long local = t - g.split_begin[s], c0 = local % quads * 4, row = local / quads;
    u64 w[4] = {0, 0, 0, 0};
    if (row < d.q) {
        const W *src = req + row / d.qpc * g.in_block + d.in_off + row % d.qpc * d.k;
#pragma unroll
        for (int b = 0; b < 4; ++b) w[b] = c0 + b < d.k ? (u64)src[c0 + b] : 0;
    }
    const long long at = spir::b_offset(row, c0, col_tiles), plane = digit_plane_of(d);
    for (int j = 0; j < spir::digits(g.ct); ++j) {
        unsigned digit = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) digit |= spir::query_digit(w[b], g.ct, j) << (8 * b);
        *reinterpret_cast<unsigned *>(d.digits + j * plane + at) = digit;
    }
}

// response_kernel over the group's flat work items: CTA blockIdx.x is one (shard, row CTA, query-tile pair, K range)
template <int D>
__global__ void __launch_bounds__(kWarps * 32) response_shards_kernel(const ShardGroup g, u64 *__restrict__ acc) {
    const long long item = blockIdx.x;
    const int s = spir::item_shard(g.item_begin, g.count, item);
    const ShardDesc &d = g.shard[s];
    const long long col_tiles = col_tiles_of(d.k);
    const spir::ItemShape shape{(d.m + spir::kCtaRows - 1) / spir::kCtaRows, (d.q + spir::kCtaQueries - 1) / spir::kCtaQueries,
                                d.split_tiles, 0};
    long long row_cta, pair, kt_begin, kt_end;
    spir::decode_item(shape, col_tiles, item - g.item_begin[s], row_cta, pair, kt_begin, kt_end);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long rt0 = (row_cta * kWarps + warp) * kWarpRowTiles;
    if (rt0 * spir::kTileRows >= d.m) return;  // padding rows only; the kernel has no block-wide barrier
    const long long qt0 = pair * kCtaQueryTiles;
    const ResponseArgs a{d.planes, d.plane_bytes, g.planes, d.digits, digit_plane_of(d), col_tiles, d.m, d.q,
                         d.split_tiles, g.ct};
    response_warp<D>(a, rt0, qt0, kt_begin, kt_end, lane, [&](long long query, long long row) {
        return acc + query / d.qpc * g.out_block + d.out_off + query % d.qpc * d.m + row;
    });
}

// responses[q][r] = acc[q][r] mod 2^ct in the reference's scalar width (query q = request * chunksPerEntry + chunk)
template <typename W>
__global__ void __launch_bounds__(kThreads) finish_kernel(const u64 *__restrict__ acc, long long words, int ct, W *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t < words) out[t] = (W)spir::finish(acc[t], ct);
}

// ---- requests and responses in protobuf messages (simple_pir.cuh, "requests and responses in protobuf messages").
// Each tile of kProtoTile virtual bytes (decode) or values (encode) is one CTA of kThreads threads, kProtoItems each.
struct ProtoRun {  // one data run: its first byte in the uploaded messages, its first virtual byte and its length
    long long src, vbegin, bytes;
};
struct DecodeMsg {  // one request message
    unsigned char *digits;           // its shard's request digit planes
    long long plane_bytes, col_tiles, columns, row_base, expected;  // expected = row_count x col_count
    long long tile_begin, run_begin;  // its first tile and run
    int word32;
};
struct EncodeMsg {  // one response message
    const u64 *acc;                  // its rows' accumulators: rows x columns, row-major
    long long rows, columns, tile_begin, tile_end;
    unsigned long long out;          // its slot in the output
};

__device__ __forceinline__ int find_last_le(const long long *begin, int count, long long key, int stride) {
    int lo = 0, hi = count - 1;  // the last i with begin[i * stride] <= key (begin[0] <= key)
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (begin[(long long)mid * stride] <= key) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// exclusive scan of one value per thread over the CTA (kThreads); total gets the CTA's sum
__device__ __forceinline__ unsigned long long block_scan(unsigned long long v, unsigned long long &total) {
    __shared__ unsigned long long warp_sums[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    unsigned long long before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        before += w < warp ? warp_sums[w] : 0;
        total += warp_sums[w];
    }
    __syncthreads();
    return before + x - v;
}

// The virtual bytes of thread threadIdx.x of tile `tile`, visited in order: f(byte pointer, run's first byte pointer,
// whether it is its run's last byte)
template <typename F>
__device__ __forceinline__ void for_each_byte(const unsigned char *msgs, const ProtoRun *runs, int run_count, int run_begin,
                                              int run_end, long long tile, F f) {
    const long long v0 = tile * spir::kProtoTile + (long long)threadIdx.x * spir::kProtoItems;
    if (run_begin >= run_end || v0 < runs[run_begin].vbegin) return;
    int r = run_begin + find_last_le(&runs[run_begin].vbegin, run_end - run_begin, v0, (int)(sizeof(ProtoRun) / 8));
    for (long long v = v0; v < v0 + spir::kProtoItems; ++v) {
        while (r < run_end && v >= runs[r].vbegin + runs[r].bytes) ++r;
        if (r >= run_end) return;
        if (v < runs[r].vbegin) continue;
        const long long off = v - runs[r].vbegin;
        f(msgs + runs[r].src + off, msgs + runs[r].src, off == runs[r].bytes - 1);
    }
}

__device__ __forceinline__ int decode_message(const DecodeMsg *m, int count, long long tile) {
    return find_last_le(&m[0].tile_begin, count, tile, (int)(sizeof(DecodeMsg) / 8));
}

// decode 1: the varints (bytes with the top bit clear) of every tile -> tile_sums[tile]
__global__ void __launch_bounds__(kThreads) proto_count_kernel(const unsigned char *__restrict__ msgs,
                                                               const ProtoRun *__restrict__ runs, int run_count,
                                                               const DecodeMsg *__restrict__ m, int count,
                                                               unsigned long long *__restrict__ tile_sums) {
    const long long tile = blockIdx.x;
    const int j = decode_message(m, count, tile);
    const int run_end = j + 1 < count ? (int)m[j + 1].run_begin : run_count;
    unsigned long long n = 0;
    for_each_byte(msgs, runs, run_count, (int)m[j].run_begin, run_end, tile,
                  [&](const unsigned char *b, const unsigned char *, bool) { n += !(*b & 0x80); });
    unsigned long long total;
    block_scan(n, total);
    if (threadIdx.x == 0) tile_sums[tile] = total;
}

// sums[0 .. n) -> their exclusive prefix sums, sums[n] = the total; one CTA of 1024 threads
__global__ void __launch_bounds__(1024) proto_scan_kernel(unsigned long long *__restrict__ sums, long long n) {
    __shared__ unsigned long long warp_sums[32];
    __shared__ unsigned long long carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    constexpr int kPer = 8;
    for (long long base = 0; base < n; base += 1024 * kPer) {
        const long long at = base + (long long)threadIdx.x * kPer;
        unsigned long long v[kPer], x = 0;
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            v[i] = at + i < n ? sums[at + i] : 0;
            x += v[i];
        }
        const unsigned long long mine = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        unsigned long long before = carry, all = carry;
        for (int w = 0; w < 32; ++w) {
            before += w < warp ? warp_sums[w] : 0;
            all += warp_sums[w];
        }
        before += x - mine;
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            if (at + i < n) sums[at + i] = before;
            before += v[i];
        }
        __syncthreads();
        if (threadIdx.x == 0) carry = all;
        __syncthreads();
    }
    if (threadIdx.x == 0) sums[n] = carry;
}

// decode 2: every varint of every tile into its shard's request digit planes (zeroed before), and the flags of the
// message it belongs to (simple_pir.cuh, ProtoFlag)
__global__ void __launch_bounds__(kThreads) proto_decode_kernel(const unsigned char *__restrict__ msgs,
                                                                const ProtoRun *__restrict__ runs, int run_count,
                                                                const DecodeMsg *__restrict__ m, int count,
                                                                const unsigned long long *__restrict__ prefix, int ct,
                                                                unsigned *__restrict__ flags) {
    const long long tile = blockIdx.x;
    const int j = decode_message(m, count, tile);
    const DecodeMsg d = m[j];
    const int run_end = j + 1 < count ? (int)m[j + 1].run_begin : run_count;
    unsigned long long n = 0;
    for_each_byte(msgs, runs, run_count, (int)d.run_begin, run_end, tile,
                  [&](const unsigned char *b, const unsigned char *, bool) { n += !(*b & 0x80); });
    unsigned long long total;
    unsigned long long index = prefix[tile] - prefix[d.tile_begin] + block_scan(n, total);
    unsigned flag = 0;
    const int digits = spir::digits(ct);
    for_each_byte(msgs, runs, run_count, (int)d.run_begin, run_end, tile,
                  [&](const unsigned char *b, const unsigned char *run, bool last) {
                      if (*b & 0x80) {
                          if (last) flag |= spir::kRunsPast;
                          return;
                      }
                      int length;
                      const uint64_t v = spir::varint_ending(run, 0, b - run, length);
                      if (length > spir::kVarintMax) flag |= spir::kLongVarint;
                      if (d.word32 && (v >> 32)) flag |= spir::kScalarRange;
                      if ((long long)index < d.expected) {
                          const long long at = spir::request_digit_at((long long)index, d.columns, d.row_base, d.col_tiles);
                          for (int k = 0; k < digits; ++k) d.digits[k * d.plane_bytes + at] = (unsigned char)spir::query_digit(v, ct, k);
                      }
                      ++index;
                  });
    if (flag) atomicOr(flags + j, flag);
}

// decode 3: each message's varint count against row_count x col_count
__global__ void __launch_bounds__(kThreads) proto_check_kernel(const DecodeMsg *__restrict__ m, int count,
                                                               long long tiles, const unsigned long long *__restrict__ prefix,
                                                               unsigned *__restrict__ flags) {
    const int j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= count) return;
    const long long end = j + 1 < count ? m[j + 1].tile_begin : tiles;
    if ((long long)(prefix[end] - prefix[m[j].tile_begin]) != m[j].expected) flags[j] |= spir::kWrongCount;
}

__device__ __forceinline__ int encode_message(const EncodeMsg *m, int count, long long tile) {
    return find_last_le(&m[0].tile_begin, count, tile, (int)(sizeof(EncodeMsg) / 8));
}

// encode 1: the varint bytes of every tile's values (acc mod 2^ct) -> tile_sums[tile]
__global__ void __launch_bounds__(kThreads) proto_length_kernel(const EncodeMsg *__restrict__ m, int count, int ct,
                                                                unsigned long long *__restrict__ tile_sums) {
    const long long tile = blockIdx.x;
    const EncodeMsg d = m[encode_message(m, count, tile)];
    const long long i0 = (tile - d.tile_begin) * spir::kProtoTile + (long long)threadIdx.x * spir::kProtoItems;
    const long long values = d.rows * d.columns;
    unsigned long long n = 0;
#pragma unroll 4
    for (int i = 0; i < spir::kProtoItems; ++i)
        if (i0 + i < values) n += spir::varint_bytes(spir::finish(d.acc[i0 + i], ct));
    unsigned long long total;
    block_scan(n, total);
    if (threadIdx.x == 0) tile_sums[tile] = total;
}

// encode 2: every message whole -- thread 0 of its first tile writes its framing and length -- and every value's
// varint after the framing
__global__ void __launch_bounds__(kThreads) proto_write_kernel(const EncodeMsg *__restrict__ m, int count, int ct,
                                                               const unsigned long long *__restrict__ prefix,
                                                               unsigned char *__restrict__ out,
                                                               unsigned long long *__restrict__ lengths) {
    const long long tile = blockIdx.x;
    const int j = encode_message(m, count, tile);
    const EncodeMsg d = m[j];
    const long long i0 = (tile - d.tile_begin) * spir::kProtoTile + (long long)threadIdx.x * spir::kProtoItems;
    const long long values = d.rows * d.columns;
    unsigned long long n = 0;
    for (int i = 0; i < spir::kProtoItems; ++i)
        if (i0 + i < values) n += spir::varint_bytes(spir::finish(d.acc[i0 + i], ct));
    unsigned long long total;
    const unsigned long long before = block_scan(n, total);
    const unsigned long long data = prefix[d.tile_end] - prefix[d.tile_begin];
    unsigned char *slot = out + d.out;
    const int header = spir::response_header(d.rows, d.columns, data, nullptr);
    if (tile == d.tile_begin && threadIdx.x == 0) {
        spir::response_header(d.rows, d.columns, data, slot);
        lengths[j] = header + data;
    }
    unsigned char *o = slot + header + (prefix[tile] - prefix[d.tile_begin]) + before;
    for (int i = 0; i < spir::kProtoItems; ++i)
        if (i0 + i < values) o += spir::put_varint(o, spir::finish(d.acc[i0 + i], ct));
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

template <int D>
cudaError_t launch_response_shards(const ShardGroup &g, long long items, u64 *acc, cudaStream_t s) {
    return launch(response_shards_kernel<D>, (unsigned)items, kWarps * 32, 0, s, g, acc);
}

// The work of a grouped response whose descriptors have their planes, m, k, q, qpc, in_off and out_off set: each
// shard's K split (desc[i].split_tiles), work items and split_shards_kernel threads, and the scratch layout -- the
// accumulators (acc_bytes), then each shard's digit planes at digit_at[i] (multiples of 512 bytes)
struct ShardPlan {
    std::vector<long long> items, split_threads;
    std::vector<size_t> digit_at;
    size_t scratch = 0;
};
ShardPlan plan_shards(std::vector<ShardDesc> &desc, size_t acc_bytes, int digits, int sms) {
    ShardPlan p;
    long long ctas = 0;
    for (const ShardDesc &d : desc) ctas += spir::base_ctas(d.m, d.q);
    p.scratch = acc_bytes;
    for (ShardDesc &d : desc) {
        const long long col_tiles = (d.k + spir::kTileCols - 1) / spir::kTileCols;
        const spir::ItemShape shape = spir::item_shape(d.m, col_tiles, d.q, ctas, sms, kMinSplitTiles);
        d.split_tiles = shape.split_tiles;
        p.items.push_back(spir::item_count(shape));
        const long long q_pad = shape.pairs * spir::kCtaQueries;
        p.split_threads.push_back(q_pad * col_tiles * (spir::kTileCols / 4));
        p.digit_at.push_back(p.scratch);
        p.scratch += (size_t)q_pad * col_tiles * spir::kTileCols * digits;
    }
    return p;
}

// The split (unless d_req is null: the digit planes are written already) and response launches of every group of
// <= kMaxShards shards of a plan, into the accumulators at the start of d_scratch
template <typename W>
cudaError_t launch_shard_groups(const std::vector<ShardDesc> &desc, const ShardPlan &plan, int planes, int ct,
                                long long in_block, long long out_block, unsigned char *d_scratch, const W *d_req,
                                cudaStream_t s) {
    const int digits = spir::digits(ct), shard_count = (int)desc.size();
    u64 *acc = reinterpret_cast<u64 *>(d_scratch);
    cudaError_t e = cudaSuccess;
    for (int first = 0, end = 0; e == cudaSuccess && first < shard_count; first = end) {
        end = spir::group_end(plan.items.data(), first, shard_count, kMaxShards, INT_MAX);
        ShardGroup g{};
        g.count = end - first;
        g.planes = planes;
        g.ct = ct;
        g.in_block = in_block;
        g.out_block = out_block;
        long long group_items = 0;
        for (int j = 0; j < g.count; ++j) {
            g.shard[j] = desc[first + j];
            g.shard[j].digits = d_scratch + plan.digit_at[first + j];
            g.item_begin[j] = group_items;
            g.split_begin[j] = g.split_threads;
            group_items += plan.items[first + j];
            g.split_threads += plan.split_threads[first + j];
        }
        if (d_req) e = launch(split_shards_kernel<W>, blocks_for(g.split_threads), kThreads, 0, s, d_req, g);
        if (e != cudaSuccess) break;
        switch (digits) {
            case 1: e = launch_response_shards<1>(g, group_items, acc, s); break;
            case 2: e = launch_response_shards<2>(g, group_items, acc, s); break;
            case 3: e = launch_response_shards<3>(g, group_items, acc, s); break;
            case 4: e = launch_response_shards<4>(g, group_items, acc, s); break;
            case 5: e = launch_response_shards<5>(g, group_items, acc, s); break;
            case 6: e = launch_response_shards<6>(g, group_items, acc, s); break;
            case 7: e = launch_response_shards<7>(g, group_items, acc, s); break;
            default: e = launch_response_shards<8>(g, group_items, acc, s); break;
        }
    }
    return e;
}

int sm_count() {
    int dev = 0, sms = 1;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

// the grouped computeResponse for `count` clients already on the device, enqueued on s: one scratch allocation, one
// memset, a split and a response launch per group of <= kMaxShards shards, one finish
template <typename W>
cudaError_t response_shards_device(const hecuda_simple_pir_database *const *shards, int shard_count, int64_t per_shard,
                                   const W *d_req, int64_t count, W *d_out, cudaStream_t s) {
    const int ct = shards[0]->params.ciphertext_modulus_bits, digits = spir::digits(ct);
    std::vector<ShardDesc> desc(shard_count);
    long long in_block = 0, out_block = 0;
    for (int i = 0; i < shard_count; ++i) {
        const hecuda_simple_pir_database &db = *shards[i];
        ShardDesc &d = desc[i];
        d.planes = db.d_planes;
        d.plane_bytes = db.plane_bytes;
        d.m = db.m;
        d.k = db.k;
        d.qpc = per_shard * db.params.chunks_per_entry;
        d.q = count * d.qpc;
        d.in_off = in_block;
        d.out_off = out_block;
        in_block += d.qpc * db.k;
        out_block += d.qpc * db.m;
    }
    const size_t acc_bytes = (size_t)count * out_block * sizeof(u64);
    const ShardPlan plan = plan_shards(desc, acc_bytes, digits, sm_count());
    unsigned char *d_scratch = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_scratch, plan.scratch, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_scratch, 0, acc_bytes, s);
    u64 *acc = reinterpret_cast<u64 *>(d_scratch);
    if (e == cudaSuccess) e = launch_shard_groups(desc, plan, shards[0]->planes, ct, in_block, out_block, d_scratch, d_req, s);
    if (e == cudaSuccess)
        e = launch(finish_kernel<W>, blocks_for(count * out_block), kThreads, 0, s, (const u64 *)acc, (long long)(count * out_block),
                   ct, d_out);
    if (d_scratch) cudaFreeAsync(d_scratch, s);
    return e;
}

// words of one client's requests (in) and responses (out) over every shard
void client_words(const hecuda_simple_pir_database *const *shards, int shard_count, int64_t per_shard, size_t &in,
                  size_t &out) {
    in = out = 0;
    for (int i = 0; i < shard_count; ++i) {
        in += (size_t)per_shard * shards[i]->params.chunks_per_entry * shards[i]->k;
        out += (size_t)per_shard * shards[i]->params.chunks_per_entry * shards[i]->m;
    }
}

int32_t check_shards(const hecuda_simple_pir_database *const *shards, int32_t shard_count, int64_t per_shard,
                     const void *req, int64_t count, const void *out) {
    if (!shards || shard_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "no shards");
    if (per_shard < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "requests_per_shard must be positive");
    if (count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative client count");
    if (count && (!req || !out)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    for (int i = 0; i < shard_count; ++i) {
        const hecuda_simple_pir_database *db = shards[i];
        if (!db) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null shard");
        if (db->params.ciphertext_modulus_bits != shards[0]->params.ciphertext_modulus_bits ||
            db->params.word_bits != shards[0]->params.word_bits)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "shards differ in ciphertextModulusBits or word_bits");
        if (db->device != shards[0]->device) return fail(HECUDA_ERR_INVALID_ARGUMENT, "shards on different devices");
        const int64_t limit = (1ll << 40) / std::max<int64_t>(1, db->params.chunks_per_entry * std::max(db->k, db->m));
        if (per_shard > limit || count > limit / per_shard)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "too many requests for one call");
    }
    return select_device(shards[0]->device);
}

// A shard's params against its rows: databaseColumns as computingParams derives it from entryCount = rows
bool columns_match(const hecuda_simple_pir_params &p, int64_t rows) {
    const int64_t epc = p.entries_per_column;
    return epc == 1 ? p.database_columns == rows * p.chunks_per_entry
                    : p.database_columns == std::max<int64_t>((rows + epc - 1) / epc, 1);
}

// ---- requests and responses in protobuf messages: the host walk of every message, then the device call
struct ProtoWalk {
    std::vector<spirproto::Request> req;
    std::vector<uint64_t> capacity;  // each response's slot
};

// Every refusal of the call, before anything is enqueued: the shards (one ct and digit-plane count, one device), then
// each message's walk, shard index, column count and size, named "message <j>: "
int32_t walk_proto_messages(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                            const uint8_t *const *messages, const uint64_t *byte_counts, int64_t count, ProtoWalk &w) {
    if (!shards || shard_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "no shards");
    if (count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative message count");
    if (count && (!messages || !byte_counts)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    for (int i = 0; i < shard_count; ++i) {
        if (!shards[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null shard");
        if (shards[i]->params.ciphertext_modulus_bits != shards[0]->params.ciphertext_modulus_bits ||
            shards[i]->planes != shards[0]->planes)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "shards differ in ciphertextModulusBits or ceil(plaintextModulusBits / 8)");
        if (shards[i]->device != shards[0]->device) return fail(HECUDA_ERR_INVALID_ARGUMENT, "shards on different devices");
    }
    const int ct = shards[0]->params.ciphertext_modulus_bits;
    w.req.assign((size_t)count, spirproto::Request{});
    w.capacity.assign((size_t)count, 0);
    std::vector<long long> rows(shard_count, 0);
    for (int64_t j = 0; j < count; ++j) {
        const std::string at = "message " + std::to_string(j) + ": ";
        if (!messages[j] && byte_counts[j]) return fail(HECUDA_ERR_INVALID_ARGUMENT, at + "null message");
        proto::Error e;
        spirproto::Request &r = w.req[(size_t)j];
        if (!spirproto::walk_request(messages[j], (long long)byte_counts[j], r, e)) return fail(e.code, at + e.what);
        if (!r.has_request) return fail(HECUDA_ERR_INVALID_ARGUMENT, at + "SimplePIRRequest.request is not set");
        if (r.shard_index >= (uint32_t)shard_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, at + "shard_index " + std::to_string(r.shard_index) + " of " +
                                                         std::to_string(shard_count) + " shards");
        const hecuda_simple_pir_database &db = *shards[r.shard_index];
        const long long R = r.matrix.rows;
        if ((int64_t)r.matrix.columns != db.k)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, at + "col_count " + std::to_string(r.matrix.columns) +
                                                         ", expected databaseColumns " + std::to_string(db.k));
        rows[r.shard_index] += R;
        if (rows[r.shard_index] > (1ll << 36) / std::max<int64_t>(1, std::max(db.k, db.m)))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, at + "row_count x col_count too large for one call");
        w.capacity[(size_t)j] = spir::response_capacity((uint64_t)R, (uint64_t)db.m, ct);
    }
    return select_device(shards[0]->device);
}

// The call after the walk: messages up once, the decode into every shard's digit planes, one grouped response over the
// shards that have rows, the encode straight from the accumulators, one download
cudaError_t response_proto(const hecuda_simple_pir_database *const *shards, int shard_count, const uint8_t *const *messages,
                           const uint64_t *byte_counts, int64_t count, const ProtoWalk &w, std::vector<unsigned char> &out,
                           std::vector<uint64_t> &slot, std::vector<unsigned long long> &lengths, std::vector<unsigned> &flags) {
    const int ct = shards[0]->params.ciphertext_modulus_bits, digits = spir::digits(ct);
    const long long T = spir::kProtoTile;
    // the shards' query blocks: message j's rows follow those of the messages before it that go to its shard
    std::vector<long long> shard_rows(shard_count, 0), row_base((size_t)count);
    for (int64_t j = 0; j < count; ++j) {
        row_base[(size_t)j] = shard_rows[w.req[(size_t)j].shard_index];
        shard_rows[w.req[(size_t)j].shard_index] += w.req[(size_t)j].matrix.rows;
    }
    std::vector<ShardDesc> desc;
    std::vector<int> slot_of(shard_count, -1);
    long long out_words = 0;
    for (int i = 0; i < shard_count; ++i) {
        if (!shard_rows[i]) continue;
        ShardDesc d{};
        d.planes = shards[i]->d_planes;
        d.plane_bytes = shards[i]->plane_bytes;
        d.m = shards[i]->m;
        d.k = shards[i]->k;
        d.q = d.qpc = shard_rows[i];
        d.out_off = out_words;
        out_words += d.q * d.m;
        slot_of[i] = (int)desc.size();
        desc.push_back(d);
    }
    const size_t acc_bytes = (size_t)out_words * sizeof(u64);
    const ShardPlan plan = plan_shards(desc, acc_bytes, digits, sm_count());
    // the messages' bytes, runs and tiles
    std::vector<ProtoRun> runs;
    std::vector<DecodeMsg> dm((size_t)count);
    std::vector<EncodeMsg> em((size_t)count);
    std::vector<long long> msg_at((size_t)count + 1, 0);
    slot.assign((size_t)count + 1, 0);
    long long tiles = 0, out_tiles = 0;
    for (int64_t j = 0; j < count; ++j) {
        const spirproto::Request &r = w.req[(size_t)j];
        const int s = (int)r.shard_index;
        const hecuda_simple_pir_database &db = *shards[s];
        msg_at[(size_t)j + 1] = msg_at[(size_t)j] + (long long)((byte_counts[j] + 15) / 16 * 16);
        DecodeMsg &d = dm[(size_t)j];
        d.digits = nullptr;  // set once the scratch is allocated
        d.col_tiles = db.col_tiles;
        d.columns = db.k;
        d.row_base = row_base[(size_t)j];
        d.expected = (long long)r.matrix.rows * (long long)r.matrix.columns;
        d.tile_begin = tiles;
        d.run_begin = (long long)runs.size();
        d.word32 = db.params.word_bits == 32;
        long long v = tiles * T;
        for (const auto &run : r.matrix.runs) {
            runs.push_back(ProtoRun{msg_at[(size_t)j] + run.first, v, run.second - run.first});
            v += run.second - run.first;
        }
        tiles += std::max<long long>(1, (v - tiles * T + T - 1) / T);
        EncodeMsg &o = em[(size_t)j];
        o.rows = r.matrix.rows;
        o.columns = db.m;
        o.tile_begin = out_tiles;
        out_tiles += std::max<long long>(1, (o.rows * o.columns + T - 1) / T);
        o.tile_end = out_tiles;
        o.out = slot[(size_t)j];
        slot[(size_t)j + 1] = slot[(size_t)j] + w.capacity[(size_t)j];
    }
    // device buffers: scratch (accumulators, digit planes), messages, runs, descriptors, sums, flags, lengths, output
    const size_t run_bytes = std::max<size_t>(1, runs.size()) * sizeof(ProtoRun);
    const size_t sum_words = (size_t)std::max(tiles, out_tiles) + 1;
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += (bytes + 255) / 256 * 256;
        return o;
    };
    const size_t o_scratch = take(plan.scratch), o_msgs = take((size_t)msg_at[(size_t)count]), o_runs = take(run_bytes),
                 o_dm = take(dm.size() * sizeof(DecodeMsg)), o_em = take(em.size() * sizeof(EncodeMsg)),
                 o_sums = take(sum_words * 8), o_flags = take((size_t)count * 4), o_len = take((size_t)count * 8),
                 o_out = take(slot[(size_t)count]);
    unsigned char *d_all = nullptr;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_all, std::max<size_t>(at, 256), s);
    unsigned char *d_scratch = d_all + o_scratch, *d_msgs = d_all + o_msgs;
    for (size_t j = 0; j < dm.size(); ++j) {
        const int k = slot_of[w.req[j].shard_index];
        if (k < 0) continue;  // no rows: nothing is decoded into it
        dm[j].digits = d_scratch + plan.digit_at[(size_t)k];
        dm[j].plane_bytes = (long long)(desc[(size_t)k].q + spir::kCtaQueries - 1) / spir::kCtaQueries * spir::kCtaQueries *
                            dm[j].col_tiles * spir::kTileCols;
        em[j].acc = reinterpret_cast<const u64 *>(d_scratch) + desc[(size_t)k].out_off + dm[j].row_base * desc[(size_t)k].m;
    }
    for (size_t j = 0; j < em.size(); ++j)
        if (!em[j].acc) em[j].acc = reinterpret_cast<const u64 *>(d_scratch);  // no values to read
    if (e == cudaSuccess) e = cudaMemsetAsync(d_scratch, 0, plan.scratch, s);
    for (int64_t j = 0; e == cudaSuccess && j < count; ++j)
        if (byte_counts[j]) e = cudaMemcpyAsync(d_msgs + msg_at[(size_t)j], messages[j], byte_counts[j], cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && !runs.empty()) e = cudaMemcpyAsync(d_all + o_runs, runs.data(), runs.size() * sizeof(ProtoRun), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_all + o_dm, dm.data(), dm.size() * sizeof(DecodeMsg), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_all + o_em, em.data(), em.size() * sizeof(EncodeMsg), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_all + o_flags, 0, (size_t)count * 4, s);
    const ProtoRun *d_runs = reinterpret_cast<const ProtoRun *>(d_all + o_runs);
    const DecodeMsg *d_dm = reinterpret_cast<const DecodeMsg *>(d_all + o_dm);
    const EncodeMsg *d_em = reinterpret_cast<const EncodeMsg *>(d_all + o_em);
    unsigned long long *d_sums = reinterpret_cast<unsigned long long *>(d_all + o_sums);
    unsigned *d_flags = reinterpret_cast<unsigned *>(d_all + o_flags);
    unsigned long long *d_len = reinterpret_cast<unsigned long long *>(d_all + o_len);
    const int n = (int)count, run_count = (int)runs.size();
    if (e == cudaSuccess)
        e = launch(proto_count_kernel, (unsigned)tiles, kThreads, 0, s, (const unsigned char *)d_msgs, d_runs, run_count, d_dm, n, d_sums);
    if (e == cudaSuccess) e = launch(proto_scan_kernel, 1, 1024, 0, s, d_sums, tiles);
    if (e == cudaSuccess)
        e = launch(proto_decode_kernel, (unsigned)tiles, kThreads, 0, s, (const unsigned char *)d_msgs, d_runs, run_count, d_dm, n,
                   (const unsigned long long *)d_sums, ct, d_flags);
    if (e == cudaSuccess)
        e = launch(proto_check_kernel, blocks_for(count), kThreads, 0, s, d_dm, n, tiles, (const unsigned long long *)d_sums, d_flags);
    if (e == cudaSuccess && !desc.empty())
        e = launch_shard_groups<u64>(desc, plan, shards[0]->planes, ct, 0, 0, d_scratch, nullptr, s);
    if (e == cudaSuccess) e = launch(proto_length_kernel, (unsigned)out_tiles, kThreads, 0, s, d_em, n, ct, d_sums);
    if (e == cudaSuccess) e = launch(proto_scan_kernel, 1, 1024, 0, s, d_sums, out_tiles);
    if (e == cudaSuccess)
        e = launch(proto_write_kernel, (unsigned)out_tiles, kThreads, 0, s, d_em, n, ct, (const unsigned long long *)d_sums,
                   d_all + o_out, d_len);
    flags.assign((size_t)count, 0);
    lengths.assign((size_t)count, 0);
    out.resize(slot[(size_t)count]);
    if (e == cudaSuccess) e = cudaMemcpyAsync(flags.data(), d_flags, (size_t)count * 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(lengths.data(), d_len, (size_t)count * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && !out.empty()) e = cudaMemcpyAsync(out.data(), d_all + o_out, out.size(), cudaMemcpyDeviceToHost, s);
    if (d_all) cudaFreeAsync(d_all, s);
    if (s) {
        const cudaError_t e2 = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(s);
    }
    return e;
}

}  // namespace

namespace hecuda {
namespace api {

int32_t simple_pir_derive(const hecuda_simple_pir_params *params, int64_t &m, int64_t &k, int64_t &entry_scalars, u64 &p) {
    Derived d;
    const int32_t rc = derive(params, d);
    if (rc) return rc;
    m = d.m, k = d.k, entry_scalars = d.entry_scalars, p = d.p;
    return HECUDA_OK;
}

}  // namespace api
}  // namespace hecuda

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

int32_t hecuda_simple_pir_process_shards(const uint8_t *values, const uint64_t *offsets, int64_t entry_count,
                                         int64_t chunk_size, int32_t shard_count, const int64_t *chunk_locations,
                                         const hecuda_simple_pir_params *params, const uint8_t *seeds, void *hints,
                                         hecuda_simple_pir_database **out) {
    if (!out || !values || !offsets || !chunk_locations || !params || !seeds || !hints)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (entry_count < 0 || shard_count < 1 || chunk_size < 1)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "entry_count, shard_count and chunk_size must be positive");
    for (int s = 0; s < shard_count; ++s) out[s] = nullptr;
    for (int64_t i = 0; i < entry_count; ++i)
        if (offsets[i + 1] < offsets[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "offsets must not decrease");
    std::vector<Derived> d(shard_count);
    for (int s = 0; s < shard_count; ++s) {
        const int32_t rc = derive(params + s, d[s]);
        if (rc) return rc;
        const hecuda_simple_pir_params &p = params[s], &p0 = params[0];
        if (p.entry_size != chunk_size) return fail(HECUDA_ERR_INVALID_ARGUMENT, "a shard's entry_size is not chunk_size");
        if (p.plaintext_modulus_bits != p0.plaintext_modulus_bits || p.ciphertext_modulus_bits != p0.ciphertext_modulus_bits ||
            p.lattice_dimension != p0.lattice_dimension || p.word_bits != p0.word_bits)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "shards differ in pt, ct, N or word_bits");
    }
    std::vector<long long> row_begin(shard_count + 1), row_source;
    {
        int64_t chunks = 0;
        for (int64_t i = 0; i < entry_count; ++i) chunks += (int64_t)((offsets[i + 1] - offsets[i] + chunk_size - 1) / chunk_size);
        row_source.resize(2 * chunks);
    }
    if (!spir::shard_rows(offsets, entry_count, chunk_size, chunk_locations, shard_count, row_begin.data(), row_source.data()))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "chunk locations are not a permutation of every shard's rows, or a shard is empty");
    for (int s = 0; s < shard_count; ++s)
        if (!columns_match(params[s], row_begin[s + 1] - row_begin[s]))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "a shard's params do not match its row count");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    std::string err;
    Context *ctx = Context::create(params[0].lattice_dimension, &d[0].p, 1, 2, err, 64);
    if (!ctx) return fail(HECUDA_ERR_UNSUPPORTED, err);
    const int64_t n = params[0].lattice_dimension;
    const bool wide = params[0].word_bits == 64;
    const size_t value_bytes = entry_count ? offsets[entry_count] : 0;
    int64_t most_rows = 0;
    for (int s = 0; s < shard_count; ++s) most_rows = std::max(most_rows, d[s].m);
    cudaStream_t st = nullptr;
    unsigned char *d_values = nullptr, *d_seeds = nullptr;
    uint64_t *d_offsets = nullptr;
    long long *d_rows = nullptr;
    u64 *d_hint = nullptr;
    u32 *d_hint32 = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_values, std::max<size_t>(1, value_bytes), st);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_offsets, (entry_count + 1) * sizeof(uint64_t), st);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_rows, row_source.size() * sizeof(long long), st);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_seeds, (size_t)shard_count * 32, st);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_hint, (size_t)most_rows * n * sizeof(u64), st);
    if (e == cudaSuccess && !wide) e = cudaMallocAsync((void **)&d_hint32, (size_t)most_rows * n * sizeof(u32), st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_values, values, value_bytes, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_offsets, offsets, (entry_count + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_rows, row_source.data(), row_source.size() * sizeof(long long), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_seeds, seeds, (size_t)shard_count * 32, cudaMemcpyHostToDevice, st);
    procdb::PirShape ps{};
    ps.entries = d_values;
    ps.offsets = d_offsets;
    ps.entry_count = entry_count;
    ps.entry_size = chunk_size;
    ps.encoded = chunk_size;
    ps.bits = params[0].plaintext_modulus_bits;
    unsigned char *hint_out = (unsigned char *)hints;
    for (int s = 0; e == cudaSuccess && s < shard_count; ++s) {
        hecuda_simple_pir_database *db = new_database(params[s], d[s]);
        if (!db) {
            e = cudaErrorMemoryAllocation;
            break;
        }
        out[s] = db;
        e = cudaMalloc(&db->d_planes, db->plane_bytes * db->planes);
        const Geometry g = d[s].g;
        if (e == cudaSuccess)
            e = launch(pack_shard_kernel, blocks_for(g.row_tiles * spir::kTileRows * g.col_tiles * (spir::kTileCols / 4)),
                       kThreads, 0, st, ps, g, (long long)d[s].padded_entry, (long long)d[s].entry_scalars,
                       (long long)(row_begin[s + 1] - row_begin[s]), (const long long *)d_rows + 2 * row_begin[s],
                       (long long)chunk_size, db->d_planes);
        if (e == cudaSuccess) e = compute_hint(*ctx, *db, d_seeds + 32 * s, d_hint, st);
        const size_t words = (size_t)d[s].m * n;
        if (e == cudaSuccess && !wide) e = launch_narrow(d_hint, d_hint32, (int64_t)words, st);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(hint_out, wide ? (const void *)d_hint : (const void *)d_hint32, words * (wide ? 8 : 4),
                                cudaMemcpyDeviceToHost, st);
        hint_out += words * (wide ? 8 : 4);
    }
    for (void *p : {(void *)d_values, (void *)d_offsets, (void *)d_rows, (void *)d_seeds, (void *)d_hint, (void *)d_hint32})
        if (p) cudaFreeAsync(p, st);
    if (st) {
        const cudaError_t e2 = cudaStreamSynchronize(st);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(st);
    }
    delete ctx;
    if (e != cudaSuccess) {
        for (int s = 0; s < shard_count; ++s) {
            hecuda_simple_pir_database_destroy(out[s]);
            out[s] = nullptr;
        }
        return cuda_fail(e, "simple_pir_process_shards");
    }
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_compute_response_shards_device(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                         int64_t requests_per_shard, const void *requests, int64_t count,
                                                         void *responses, void *stream) {
    int32_t rc = check_shards(shards, shard_count, requests_per_shard, requests, count, responses);
    if (rc || count == 0) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e =
        shards[0]->params.word_bits == 64
            ? response_shards_device(shards, shard_count, requests_per_shard, (const u64 *)requests, count, (u64 *)responses, s)
            : response_shards_device(shards, shard_count, requests_per_shard, (const u32 *)requests, count, (u32 *)responses, s);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_compute_response_shards_device");
}

int32_t hecuda_simple_pir_compute_response_shards(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                  int64_t requests_per_shard, const void *requests, int64_t count,
                                                  void *responses) {
    int32_t rc = check_shards(shards, shard_count, requests_per_shard, requests, count, responses);
    if (rc || count == 0) return rc;
    const size_t word = shards[0]->params.word_bits / 8;
    size_t in_words = 0, out_words = 0;
    client_words(shards, shard_count, requests_per_shard, in_words, out_words);
    const size_t in_bytes = (size_t)count * in_words * word, out_bytes = (size_t)count * out_words * word;
    cudaStream_t s = nullptr;
    void *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_in, in_bytes, s);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_out, out_bytes, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, requests, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess)
        e = word == 8 ? response_shards_device(shards, shard_count, requests_per_shard, (const u64 *)d_in, count, (u64 *)d_out, s)
                      : response_shards_device(shards, shard_count, requests_per_shard, (const u32 *)d_in, count, (u32 *)d_out, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(responses, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
    for (void *p : {d_in, d_out})
        if (p) cudaFreeAsync(p, s);
    if (s) {
        const cudaError_t e2 = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = e2;
        cudaStreamDestroy(s);
    }
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "simple_pir_compute_response_shards");
}

int32_t hecuda_simple_pir_response_proto_byte_count(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                    const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                    int64_t count, uint64_t *capacities) {
    if (count && !capacities) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    ProtoWalk w;
    const int32_t rc = walk_proto_messages(shards, shard_count, messages, message_byte_counts, count, w);
    if (rc) return rc;
    std::copy(w.capacity.begin(), w.capacity.end(), capacities);
    return HECUDA_OK;
}

int32_t hecuda_simple_pir_compute_response_proto(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                 const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                 int64_t count, uint8_t *out, const uint64_t *out_offsets,
                                                 uint64_t *out_lengths) {
    if (count && (!out || !out_offsets || !out_lengths)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    ProtoWalk w;
    int32_t rc = walk_proto_messages(shards, shard_count, messages, message_byte_counts, count, w);
    if (rc || count == 0) return rc;
    for (int64_t j = 0; j + 1 < count; ++j)
        if (out_offsets[j] + w.capacity[(size_t)j] > out_offsets[j + 1])
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "message " + std::to_string(j) + ": its slot of " +
                                                         std::to_string(out_offsets[j + 1] - std::min(out_offsets[j + 1], out_offsets[j])) +
                                                         " bytes is below its capacity " + std::to_string(w.capacity[(size_t)j]));
    std::vector<unsigned char> bytes;
    std::vector<uint64_t> slot;
    std::vector<unsigned long long> lengths;
    std::vector<unsigned> flags;
    const cudaError_t e = response_proto(shards, shard_count, messages, message_byte_counts, count, w, bytes, slot, lengths, flags);
    if (e != cudaSuccess) return cuda_fail(e, "simple_pir_compute_response_proto");
    for (int64_t j = 0; j < count; ++j) {
        const unsigned f = flags[(size_t)j];
        if (!f) continue;
        std::string what = "message " + std::to_string(j) + ": ";
        if (f & spir::kLongVarint) what += "malformedProtobuf(SimplePIRMatrix.data: a varint longer than 10 bytes)";
        else if (f & spir::kRunsPast) what += "truncated(SimplePIRMatrix.data: a varint runs past the end)";
        else if (f & spir::kScalarRange) what += "SimplePIRMatrix.data: a value at or above 2^32 for a 32-bit shard";
        else what += "SimplePIRMatrix.data: the varint count is not row_count x col_count";
        return fail(HECUDA_ERR_INVALID_ARGUMENT, what);
    }
    for (int64_t j = 0; j < count; ++j) {
        std::memcpy(out + out_offsets[j], bytes.data() + slot[(size_t)j], lengths[(size_t)j]);
        out_lengths[j] = lengths[(size_t)j];
    }
    return HECUDA_OK;
}

}  // extern "C"
