// simple_pir.cuh -- the arithmetic and index maps of the SimplePIR kernels (simple_pir.cu).  Every function is __host__
// __device__, so tests/emu/simple_pir_emulate.cu replays exactly what the kernels compute on the CPU.
//
//   SimplePirServer.process            SimplePir/SimplePir+Database.swift:252-290
//   SimplePirServer.computeResponse    SimplePir/SimplePir+Server.swift:31-38, Array2d.multiply(transposing:mask:)
//                                      SimplePir+Precompute.swift:51-114
//
// The response is (DB' . request^T) mod 2^ct with DB' (M x K) below 2^pt and request words of any width.  Both sides
// are split into u8 digits: DB' into ceil(pt / 8) planes, requests (masked to ct bits first) into ceil(ct / 8) digits.
// Each (plane i, digit j) pair is one u8 x u8 -> s32 integer MMA product, summed over K-slices of at most
// kSliceColumns columns: 255 * 255 * 32768 = 2 130 739 200 < 2^31, so an s32 slice sum never saturates or wraps.  Each
// slice sum is widened into a 64-bit accumulator shifted by 8 (i + j) (mod 2^64); a pair with 8 (i + j) >= ct adds a
// multiple of 2^ct and is skipped.  Masking the 64-bit sum to ct <= 61 bits gives the reference's wrapped product.
#pragma once
#include <cstdint>

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

}  // namespace spir
}  // namespace hecuda
