// simple_pir.cuh -- the arithmetic and index maps of the SimplePIR kernels (simple_pir.cu).  Every function is __host__
// __device__, so tests/emu/simple_pir_emulate.cu, simple_pir_shards_emulate.cu and simple_pir_client_emulate.cu replay
// exactly what the kernels (simple_pir.cu, simple_pir_client.cu) compute on the CPU.
//
//   SimplePirServer.process            SimplePir/SimplePir+Database.swift:252-290
//   SimplePirServer.computeResponse    SimplePir/SimplePir+Server.swift:31-38, Array2d.multiply(transposing:mask:)
//                                      SimplePir+Precompute.swift:51-114
//   DatabaseMap.shardDatabase          SimplePir/DatabaseMap.swift:82-110
//   grouped responses over shards      SimplePir/SimplePir+Shards.swift:47-173 (one request set per shard and client)
//
// The response is (DB' . request^T) mod 2^ct with DB' (M x K) below 2^pt and request words of any width.  Both sides
// are split into u8 digits: DB' into ceil(pt / 8) planes, requests (masked to ct bits first) into ceil(ct / 8) digits.
// Each (plane i, digit j) pair is one u8 x u8 -> s32 integer MMA product, summed over K-slices of at most
// kSliceColumns columns: 255 * 255 * 32768 = 2 130 739 200 < 2^31, so an s32 slice sum never saturates or wraps.  Each
// slice sum is widened into a 64-bit accumulator shifted by 8 (i + j) (mod 2^64); a pair with 8 (i + j) >= ct adds a
// multiple of 2^ct and is skipped.  Masking the 64-bit sum to ct <= 61 bits gives the reference's wrapped product.
#pragma once
#include <cstdint>

#include "process_db.cuh"

#ifdef __CUDACC__
#define SPIR_HD __host__ __device__ __forceinline__
#else
#define SPIR_HD inline
#endif

namespace hecuda {
namespace spir {

constexpr int kSliceColumns = 32768;           // columns per s32 slice sum
constexpr int kTileRows = 16, kTileCols = 32;  // mma m16n8k32: A tile 16 rows x 32 columns
constexpr int kTileQueries = 8;                // n = 8 queries per B tile
constexpr int kSliceTiles = kSliceColumns / kTileCols;

SPIR_HD int digits(int bits) { return (bits + 7) / 8; }
SPIR_HD uint64_t low_mask(int bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1); }

// digit i of a DB' value (< 2^pt)
SPIR_HD unsigned db_digit(uint64_t v, int i) { return (unsigned)(v >> (8 * i)) & 0xffu; }
// digit j of a request word: bits at or above ct do not reach the masked result, so they are dropped first
SPIR_HD unsigned query_digit(uint64_t w, int ct, int j) { return (unsigned)((w & low_mask(ct)) >> (8 * j)) & 0xffu; }
// whether pair (i, j) can change the result mod 2^ct
SPIR_HD bool pair_live(int i, int j, int ct) { return 8 * (i + j) < ct; }
// one slice sum (as s32 bits, non-negative and < 2^31) into the 64-bit accumulator, shifted by 8 (i + j), mod 2^64
SPIR_HD uint64_t widen(uint64_t acc, uint32_t slice_sum, int i, int j) {
    const int shift = 8 * (i + j);
    return shift >= 64 ? acc : acc + ((uint64_t)slice_sum << shift);
}
SPIR_HD uint64_t finish(uint64_t acc, int ct) { return acc & low_mask(ct); }

// Resident digit plane: DB' padded to rows_pad (multiple of 16 x kRowTilesPerCta) x cols_pad (multiple of 32), cut into
// 16 x 32 tiles stored row-tile-major; inside a tile, lane l's 16 bytes are its four A-fragment registers of
// mma.m16n8k32 (a0: row g, columns 4t..4t+3; a1: row g + 8; a2, a3: the same at column 16 + 4t; g = l / 4, t = l % 4).
// One warp loads a whole tile with one coalesced 16-byte load per lane.
SPIR_HD long long a_offset(long long r, long long c, long long col_tiles) {
    const long long tile = (r / kTileRows) * col_tiles + c / kTileCols;
    const int rr = (int)(r % kTileRows), cc = (int)(c % kTileCols);
    const int lane = (rr & 7) * 4 + ((cc & 15) >> 2);
    const int reg = (cc >> 4) * 2 + (rr >> 3);
    return tile * 512 + lane * 16 + reg * 4 + (cc & 3);
}
// Request digit plane: queries padded to q_pad (multiple of 16) x cols_pad, in 8 x 32 tiles, query-tile-major; lane l's
// 8 bytes are its two B-fragment registers (b0: query g, columns 4t..4t+3; b1: columns 16 + 4t..).
SPIR_HD long long b_offset(long long q, long long c, long long col_tiles) {
    const long long tile = (q / kTileQueries) * col_tiles + c / kTileCols;
    const int cc = (int)(c % kTileCols);
    const int lane = (int)(q % kTileQueries) * 4 + ((cc & 15) >> 2);
    return tile * 256 + lane * 8 + (cc >> 4) * 4 + (cc & 3);
}

#ifdef __CUDACC__
// The warp-level u8 x u8 -> s32 MMA of the response kernels and the client's results product: c += a (16 x 32 A
// fragment, a_offset layout) . b (32 x 8 B fragment, b_offset layout)
__device__ __forceinline__ void mma_u8(int (&c)[4], const uint4 &a, const uint2 &b) {
    asm volatile(
        "mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b.x), "r"(b.y));
}
#endif

// The processed database before its transpose is row-major K x M with entry e's coefficients at e * padded_entry
// (:262-280); DB'[r][c] is its element c * M + r.  -> (entry, coefficient index), or entry = -1 for a zero.
SPIR_HD void db_source(long long r, long long c, long long m, long long padded_entry, long long entry_scalars,
                       long long entry_count, long long &entry, long long &k) {
    const long long f = c * m + r;
    entry = f / padded_entry;
    k = f - entry * padded_entry;
    if (entry >= entry_count || k >= entry_scalars) entry = -1;
}

// sigma(a) = a(x^-1) in Coeff form: sigma(a)_0 = a_0, sigma(a)_{N-i} = -a_i.  Coefficient i of a lands at sigma_index.
SPIR_HD long long sigma_index(long long i, long long n) { return i ? n - i : 0; }
SPIR_HD uint64_t sigma_value(uint64_t v, long long i, uint64_t p) { return (i && v) ? p - v : v; }

// ---- sharding: DatabaseMap.shardDatabase (SimplePir/DatabaseMap.swift:82-110)
// Entry e is cut into ceil(size / chunk_size) chunks; chunk c is bytes [c * chunk_size, (c + 1) * chunk_size) of the
// entry, zero-padded to chunk_size.  The caller's chunk locations (shard, index), entry-major, place every chunk on one
// row of one shard.  shard_rows inverts them: row_source[row_begin[s] + index] = {entry, chunk}, with row_begin the
// prefix of the shards' row counts (shard_count + 1).  Returns false, leaving row_source partly written, unless the
// locations are a permutation of every shard's rows and no shard is empty.
inline bool shard_rows(const uint64_t *offsets, long long entry_count, long long chunk_size, const int64_t *locations,
                       int shard_count, long long *row_begin, long long *row_source) {
    for (int s = 0; s <= shard_count; ++s) row_begin[s] = 0;
    long long chunks = 0;
    for (long long e = 0; e < entry_count; ++e) {
        const long long n = (long long)((offsets[e + 1] - offsets[e] + chunk_size - 1) / chunk_size);
        for (long long c = 0; c < n; ++c, ++chunks) {
            const int64_t s = locations[2 * chunks];
            if (s < 0 || s >= shard_count) return false;
            ++row_begin[s + 1];
        }
    }
    for (int s = 0; s < shard_count; ++s) {
        if (row_begin[s + 1] == 0) return false;
        row_begin[s + 1] += row_begin[s];
    }
    for (long long r = 0; r < chunks; ++r) row_source[2 * r] = -1;
    chunks = 0;
    for (long long e = 0; e < entry_count; ++e) {
        const long long n = (long long)((offsets[e + 1] - offsets[e] + chunk_size - 1) / chunk_size);
        for (long long c = 0; c < n; ++c, ++chunks) {
            const int64_t s = locations[2 * chunks], i = locations[2 * chunks + 1];
            if (i < 0 || i >= row_begin[s + 1] - row_begin[s] || row_source[2 * (row_begin[s] + i)] >= 0) return false;
            row_source[2 * (row_begin[s] + i)] = e;
            row_source[2 * (row_begin[s] + i) + 1] = c;
        }
    }
    return true;
}

// A shard's row {entry, chunk} as the bytes of the entry it holds: the chunk's bytes, shorter than chunk_size for the
// entry's last chunk; bytesToCoefficients reads the missing bytes as the zero padding shardDatabase appends.
SPIR_HD procdb::PirPiece shard_piece(const procdb::PirShape &s, long long entry, long long chunk, long long chunk_size) {
    const long long start = chunk * chunk_size, left = procdb::pir_entry_length(s, entry) - start;
    return procdb::PirPiece{entry, start, left < chunk_size ? left : chunk_size};
}

// ---- grouped responses over shards: one launch answers the queries of up to kMaxShards shards.  Its CTAs are a flat
// list of work items; shard s owns items [item_begin[s], item_begin[s] + item_count) of the launch, ordered as
// response_kernel's grid (row-CTA fastest, then query-tile pair, then K range).  A CTA covers kCtaRows rows and
// kCtaQueries queries.
constexpr int kCtaRows = 128, kCtaQueries = 16;

struct ItemShape {
    long long row_ctas, pairs;  // ceil(M / kCtaRows), padded queries / kCtaQueries
    long long split_tiles;      // 32-column tiles per K range
    long long splits;           // K ranges
};

SPIR_HD long long base_ctas(long long m, long long q) {
    return (m + kCtaRows - 1) / kCtaRows * ((q + kCtaQueries - 1) / kCtaQueries);
}
// The K split of one shard when the shards of the call make `ctas` CTAs before splitting: as response_kernel's, ranges
// until the launch covers the SMs about four times over, each of at least min_split_tiles tiles.
SPIR_HD ItemShape item_shape(long long m, long long col_tiles, long long q, long long ctas, int sm_count,
                             int min_split_tiles) {
    ItemShape s;
    s.row_ctas = (m + kCtaRows - 1) / kCtaRows;
    s.pairs = (q + kCtaQueries - 1) / kCtaQueries;
    long long splits = (4ll * sm_count + ctas - 1) / ctas;
    const long long most = col_tiles / min_split_tiles;
    splits = splits < 1 ? 1 : splits;
    splits = splits < most ? splits : (most < 1 ? 1 : most);
    s.split_tiles = (col_tiles + splits - 1) / splits;
    s.splits = (col_tiles + s.split_tiles - 1) / s.split_tiles;
    return s;
}
SPIR_HD long long item_count(const ItemShape &s) { return s.row_ctas * s.pairs * s.splits; }

// The shards [first, end) of one launch: at most max_shards, and at most max_items items unless one shard alone has more
// (the caller refuses that).  items[s] = item_count of shard s.
SPIR_HD int group_end(const long long *items, int first, int shard_count, int max_shards, long long max_items) {
    int end = first + 1;
    long long total = items[first];
    while (end < shard_count && end - first < max_shards && total + items[end] <= max_items) total += items[end++];
    return end;
}

// Item `item` of a launch whose shards start at item_begin[0..count) (ascending, item_begin[0] = 0) -> its shard, row
// CTA, query-tile pair and K range [k_begin, k_end) in 32-column tiles.
SPIR_HD int item_shard(const long long *item_begin, int count, long long item) {
    int lo = 0, hi = count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (item_begin[mid] <= item) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
SPIR_HD void decode_item(const ItemShape &s, long long col_tiles, long long local, long long &row_cta, long long &pair,
                         long long &k_begin, long long &k_end) {
    row_cta = local % s.row_ctas;
    const long long t = local / s.row_ctas;
    pair = t % s.pairs;
    k_begin = t / s.pairs * s.split_tiles;
    k_end = k_begin + s.split_tiles < col_tiles ? k_begin + s.split_tiles : col_tiles;
}

// ---- requests and responses in protobuf messages (simple_pir.cu, "proto"; the host walk is simple_pir_proto.hpp).
// A call's data runs are laid end to end in one virtual byte stream, each message's first run starting at a multiple of
// kProtoTile, so every tile belongs to one message.  A byte whose top bit is clear ends a varint; the varint's index in
// its message is the number of such bytes before it in the message's runs (a scan over tiles, then inside the tile).
// The responses' values are laid out the same way, with one tile at least per message so that empty messages get their
// framing.
constexpr int kProtoItems = 16;                      // bytes (decode) or values (encode) per thread
constexpr long long kProtoTile = 256 * kProtoItems;  // per CTA of 256 threads
constexpr int kVarintMax = 10;

SPIR_HD int varint_bytes(uint64_t v) {
    int n = 1;
    while (v >>= 7) ++n;
    return n;
}
SPIR_HD int put_varint(unsigned char *out, uint64_t v) {
    int n = 0;
    while (v >= 0x80) {
        out[n++] = (unsigned char)(v | 0x80);
        v >>= 7;
    }
    out[n++] = (unsigned char)v;
    return n;
}
// The varint ending at b[p] (its last byte) that starts after b[lo - 1]: its value, as proto::read_varint reads it
// (bits past 64 in a tenth byte are dropped), and its length; length > kVarintMax when the kVarintMax bytes before b[p]
// all carry the continuation bit, which read_varint refuses.
SPIR_HD uint64_t varint_ending(const unsigned char *b, long long lo, long long p, int &length) {
    long long s = p;
    while (s > lo && (b[s - 1] & 0x80) && p - s < kVarintMax) --s;
    length = (int)(p - s + 1);
    uint64_t v = 0;
    for (long long k = s; k <= p && k - s < kVarintMax; ++k) v |= (uint64_t)(b[k] & 0x7f) << (7 * (k - s));
    return v;
}
// Where varint `index` of a message with `columns` columns goes in its shard's request digit planes: query
// row_base + index / columns, column index % columns (b_offset)
SPIR_HD long long request_digit_at(long long index, long long columns, long long row_base, long long col_tiles) {
    return b_offset(row_base + index / columns, index % columns, col_tiles);
}
// The flags of a message the decode refuses
enum ProtoFlag : unsigned { kLongVarint = 1, kRunsPast = 2, kScalarRange = 4, kWrongCount = 8 };

// A SimplePIRResponse of rows x columns values whose data varints take data_len bytes, as SwiftProtobuf writes it:
// 0x0a len { [0x08 rows]  0x10 columns  [0x1a data_len data] } -> the framing's length; written to out unless null.
// proto3 omits a zero row count and an empty data field; the response message is written even when empty.
SPIR_HD int response_header(uint64_t rows, uint64_t columns, uint64_t data_len, unsigned char *out) {
    const uint64_t values = rows * columns;
    const uint64_t body = (rows ? 1 + varint_bytes(rows) : 0) + (columns ? 1 + varint_bytes(columns) : 0) +
                          (values ? 1 + varint_bytes(data_len) + data_len : 0);
    if (!out) return (int)(1 + varint_bytes(body) + body - (values ? data_len : 0));
    unsigned char *o = out;
    int n = 0;
    o[n++] = 0x0a;
    n += put_varint(o + n, body);
    if (rows) o[n++] = 0x08, n += put_varint(o + n, rows);
    if (columns) o[n++] = 0x10, n += put_varint(o + n, columns);
    if (values) o[n++] = 0x1a, n += put_varint(o + n, data_len);
    return n;
}
// The most bytes a response of rows x columns values below 2^ct can take: every varint ceil(ct / 7) bytes long
SPIR_HD uint64_t response_capacity(uint64_t rows, uint64_t columns, int ct) {
    const uint64_t data = rows * columns * (uint64_t)((ct + 6) / 7);
    return (uint64_t)response_header(rows, columns, data, nullptr) + (rows * columns ? data : 0);
}

// ---- the client (simple_pir_client.cu): PrecomputedQueries.WithoutIndices.init, add(index:), integrate
//   generateSecretPolys / noiselessSample / encryptZero / extractEntries   SimplePir+Client.swift:20-95
//   Array2d.multiply(transposing:modulus:)                                  SimplePir+Precompute.swift:122-188
//   Array2d.divideAndRound, randomCenteredBinomialDistribution              Array2d.swift:382-429, 489-514
// A query's secret seed draws its chunksPerEntry ternary polynomials one after another from one stream; its error seed
// draws the 1 x (chunksPerEntry K) error array, which is then read as chunksPerEntry x K.  -> stream coefficient index.
SPIR_HD long long secret_coefficient(long long i, long long j, long long n) { return i * n + j; }
SPIR_HD long long error_coefficient(long long i, long long c, long long k) { return i * k + c; }
// add(index:): the column of query row i (< chunksPerEntry) that gets delta = 2^(ct - pt)
SPIR_HD long long delta_column(long long index, long long i, long long cpe, long long epc) { return (index * cpe + i) / epc; }
// extractEntries: element t (< chunkSize) of row i of the extracted cpe x chunkSize array, as an offset into one query's
// cpe x M array (responses or resultsWithoutResponse)
SPIR_HD long long extract_offset(long long index, long long i, long long t, long long cpe, long long epc, long long m,
                                 long long chunk) {
    return i * m + (index * cpe + i) % epc * chunk + t;
}

typedef unsigned __int128 spir_u128;
SPIR_HD uint64_t mulhi(uint64_t a, uint64_t b) { return (uint64_t)(((spir_u128)a * b) >> 64); }
// floor(x / p) for any 128-bit x with the quotient below 2^64, and x mod p: Barrett with mu = floor(2^128 / p) = (mu_hi,
// mu_lo) (p < 2^63, not a power of two) gives the low word of a quotient at most 2 below the true one, then corrections
SPIR_HD uint64_t div_mod(spir_u128 x, uint64_t p, uint64_t mu_hi, uint64_t mu_lo, uint64_t &rem) {
    const uint64_t lo = (uint64_t)x, hi = (uint64_t)(x >> 64);
    const spir_u128 mid = (spir_u128)mulhi(lo, mu_lo) + (uint64_t)(lo * mu_hi) + (uint64_t)(hi * mu_lo);
    uint64_t q = hi * mu_hi + mulhi(lo, mu_hi) + mulhi(hi, mu_lo) + (uint64_t)(mid >> 64);
    uint64_t r = lo - q * p;  // the true remainder plus at most 2p, below 2^64
    for (int i = 0; i < 2; ++i)
        if (r >= p) r -= p, ++q;
    rem = r;
    return q;
}
// divideAndRound(initialMod: p, newMod: 2^ct) of x < p: floor((x 2^ct + floor(p / 2)) / p) mod 2^ct, exactly
SPIR_HD uint64_t divide_and_round(uint64_t x, uint64_t p, uint64_t mu_hi, uint64_t mu_lo, int ct) {
    uint64_t rem;
    return div_mod(((spir_u128)x << ct) + (p >> 1), p, mu_hi, mu_lo, rem) & low_mask(ct);
}
// resultsWithoutResponse = S . hint^T mod p, with the secrets stored mod p (-1 as p - 1) and the reference's sum taken
// in T.DoubleWidth with &+= (2 word_bits bits, wrapping).  With hint words split into u8 digits h = sum_d h_d 2^(8d)
// and P_d, Nn_d the digit-d sums over the secret's +1 and -1 positions, the reference's sum is
// U = sum_d (P_d + (p - 1) Nn_d) 2^(8d) mod 2^(2 word_bits).  results_add adds plane d's term mod 2^128 (a multiple of
// 2^(2 word_bits)); results_word takes U mod p.
SPIR_HD spir_u128 results_add(spir_u128 acc, uint32_t pos, uint32_t neg, int d, uint64_t p) {
    return acc + (((spir_u128)pos + (spir_u128)(p - 1) * neg) << (8 * d));
}
SPIR_HD uint64_t results_word(spir_u128 acc, int word_bits, uint64_t p, uint64_t mu_hi, uint64_t mu_lo) {
    if (word_bits == 32) acc = (uint64_t)acc;
    uint64_t rem;
    div_mod(acc, p, mu_hi, mu_lo, rem);
    return rem;
}
// integrate: ((response - result + delta / 2) & mask) >> (ct - pt), in the scalar's wrapping arithmetic (the mask keeps
// ct < word_bits bits, so 64-bit wrapping gives the same value)
SPIR_HD uint64_t integrate(uint64_t response, uint64_t result, int pt, int ct) {
    return ((response - result + ((1ull << (ct - pt)) >> 1)) & low_mask(ct)) >> (ct - pt);
}

}  // namespace spir
}  // namespace hecuda
