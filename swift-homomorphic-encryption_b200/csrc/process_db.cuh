// process_db.cuh -- index maps of the database-processing kernels (process_db.cu).  Every function is __host__
// __device__, so tests/emu/process_db_emulate.cu replays exactly what the kernels compute on the CPU.
//
//   MulPirServer.process: processPackEntries / processSplitLargeEntries   IndexPir/MulPir.swift:433-556
//   CoefficientPacking.bytesToCoefficients                                  HomomorphicEncryption/CoefficientPacking.swift
//   PlaintextMatrix.init(signedValues:) + diagonalPlaintexts                PlaintextMatrix.swift:155-190, 417-482
#pragma once
#include <math.h>

#include <cstdint>

#ifdef __CUDACC__
#define PDB_HD __host__ __device__ __forceinline__
#else
#define PDB_HD inline
#endif

namespace hecuda {
namespace procdb {

// ---- MulPir -------------------------------------------------------------------------------------------------------
// A database as MulPirServer.process sees it.  Entry i is the bytes [offsets[i], offsets[i + 1]) of `entries`, or
// [i * entry_size, (i + 1) * entry_size) without offsets.  Its encoded form is the `width`-byte little-endian length
// prefix, the entry, then zero padding up to `encoded` bytes.
struct PirShape {
    const unsigned char *entries;
    const uint64_t *offsets;  // entry_count + 1, or null
    long long entry_count, entry_size;
    long long encoded;     // IndexPirParameter.encodedEntrySize = width + entry_size
    long long capacity;    // bytesPerPlaintext = N * bits / 8
    long long stride;      // processPackEntries: bytes per plaintext, capacity / encoded * encoded; 0 = split entries
    long long per_chunk;   // prod(dimensions)
    long long dim0;        // dimensions[0]
    int width;             // entrySizeEncodingWidth (0 without encodingEntrySize)
    int bits;              // floor(log2 t) bits per coefficient
};

// The bytes one plaintext holds: `length` bytes from byte `start` of the encoded stream.  Packed entries: the
// concatenation of every encoded entry (entry = -1).  Split entries: entry `entry`'s prefix and bytes only.
// length 0 = a nil plaintext.
struct PirPiece {
    long long entry, start, length;
};

// The shape of a database (without its pointers) for a context of degree n and plaintext modulus t:
// IndexPirParameter.encodedEntrySize, bytesPerPlaintext, and the packing path (MulPir.swift:433-450).
PDB_HD PirShape pir_shape(long long n, uint64_t t, long long entry_count, long long entry_size, bool encode_entry_size,
                          long long per_chunk, long long dim0) {
    PirShape s{};
    int bits = 63;
    while (bits > 0 && !(t >> bits)) --bits;  // floor(log2 t)
    s.bits = bits;
    s.entry_count = entry_count;
    s.entry_size = entry_size;
    s.width = !encode_entry_size ? 0 : entry_size < (1ll << 8) ? 1 : entry_size < (1ll << 16) ? 2 : entry_size < (1ll << 32) ? 4 : 8;
    s.encoded = s.width + entry_size;
    s.capacity = n * bits / 8;
    s.per_chunk = per_chunk;
    s.dim0 = dim0;
    s.stride = s.capacity >= s.encoded ? s.capacity / s.encoded * s.encoded : 0;
    return s;
}
// chunkCount: plaintexts per entry (1 when entries are packed)
PDB_HD long long pir_chunk_count(const PirShape &s) { return (s.encoded + s.capacity - 1) / s.capacity; }

PDB_HD long long pir_entry_start(const PirShape &s, long long e) {
    return s.offsets ? (long long)s.offsets[e] : e * s.entry_size;
}
PDB_HD long long pir_entry_length(const PirShape &s, long long e) {
    return s.offsets ? (long long)(s.offsets[e + 1] - s.offsets[e]) : s.entry_size;
}

// Plaintext `index` in process order (chunk-major, then column-major over the first dimension) -> its piece.
PDB_HD PirPiece pir_piece(const PirShape &s, long long index) {
    const long long chunk = index / s.per_chunk, k = index - chunk * s.per_chunk;
    const long long columns = s.per_chunk / s.dim0;
    const long long row = (k % s.dim0) * columns + k / s.dim0;
    if (s.stride) {  // processPackEntries: the encoded stream cut every `stride` bytes, the last piece shorter
        const long long start = row * s.stride, total = s.entry_count * s.encoded;
        const long long left = total - start;
        return {-1, start, left <= 0 ? 0 : (left < s.stride ? left : s.stride)};
    }
    // processSplitLargeEntries: chunk k is [k * capacity - width, (k + 1) * capacity - width) of the entry, with the
    // prefix in chunk 0 -- bytes [lo, hi) of prefix + entry; a chunk past the entry's end is nil
    if (row >= s.entry_count) return {row, 0, 0};
    const long long len = pir_entry_length(s, row), lo = chunk * s.capacity;
    const long long end = lo - s.width + s.capacity;
    const long long hi = (end < len ? end : len) + s.width;
    return {row, lo, hi > lo ? hi - lo : 0};
}

// Byte j (< piece.length) of a piece: a prefix byte, an entry byte or a pad byte.
PDB_HD unsigned pir_piece_byte(const PirShape &s, const PirPiece &p, long long j) {
    long long e = p.entry, at = p.start + j;
    if (e < 0) {
        e = at / s.encoded;
        at -= e * s.encoded;
    }
    const long long len = pir_entry_length(s, e);
    if (at < s.width) return (unsigned)(((unsigned long long)len >> (8 * at)) & 0xff);
    at -= s.width;
    return at < len ? s.entries[pir_entry_start(s, e) + at] : 0u;
}

// bytesToCoefficients: coefficient i is bits [i * bits, (i + 1) * bits) of the piece's big-endian bit stream,
// zero-padded to a whole coefficient; coefficients past ceil(8 * length / bits) are 0.
PDB_HD uint64_t pir_coefficient(const PirShape &s, const PirPiece &p, long long i) {
    const long long bit = i * s.bits;
    if (bit >= 8 * p.length) return 0;
    const long long first = bit >> 3;
    const int shift = (int)(bit & 7), bytes = (shift + s.bits + 7) >> 3;
    unsigned __int128 acc = 0;
    for (int k = 0; k < bytes; ++k) {
        const long long at = first + k;
        acc = (acc << 8) | (unsigned __int128)(at < p.length ? pir_piece_byte(s, p, at) : 0u);
    }
    const uint64_t mask = s.bits >= 64 ? ~0ull : ((1ull << s.bits) - 1);
    return (uint64_t)(acc >> (8 * bytes - shift - s.bits)) & mask;
}

// coefficientsToBytes (CoefficientPacking.swift:141-217), the inverse map: byte b is bits [8b, 8b + 8) of the big-endian
// bit stream of `count` coefficients of `bits` bits each (coefficient(i) < 2^bits), zero past the last coefficient.
template <typename Coefficient>
PDB_HD unsigned coefficients_byte(Coefficient coefficient, long long count, int bits, long long b) {
    unsigned out = 0;
    long long cached = -1;
    uint64_t c = 0;
    for (int k = 0; k < 8; ++k) {
        const long long bit = 8 * b + k, i = bit / bits;
        if (i != cached && i < count) c = coefficient(i), cached = i;
        out = (out << 1) | (i < count ? (unsigned)(c >> (bits - 1 - (int)(bit - i * bits))) & 1u : 0u);
    }
    return out;
}

// ---- PNNS ---------------------------------------------------------------------------------------------------------
// A row-major rows x cols matrix in .diagonal packing: dimension = nextPow2(cols) diagonals of `results` =
// ceil(rows / N) chunks each, diagonal d's chunks rotated by floor(d / baby) * baby in both SIMD half-rows.
struct PnnsShape {
    long long rows, cols, results;
    int dimension, baby, giant, logn;
};

// Slot `slot` (0 .. N) of chunk r of diagonal d -> index of the matrix element it holds, -1 for a zero.
// Diagonal d holds data[c][(c + d) mod dimension] (0 past cols) for every database row c (0 past rows).
PDB_HD long long pnns_element(const PnnsShape &s, int d, long long r, int slot) {
    const int half = 1 << (s.logn - 1);
    const int step = d / s.baby * s.baby;
    const int h = slot & half, pos = slot & (half - 1);
    const long long c = (r << s.logn) + h + ((pos - step) & (half - 1));  // both half-rows rolled by `step`
    if (c >= s.rows) return -1;
    const long long col = (c + d) & (s.dimension - 1);
    return col < s.cols ? c * s.cols + col : -1;
}

// diagonalPlaintexts order: plaintext p is chunk p mod results of diagonal p / results
PDB_HD void pnns_plaintext(const PnnsShape &s, long long p, int &d, long long &r) {
    d = (int)(p / s.results);
    r = p - (long long)d * s.results;
}

// The resident order of hecuda_pnns_matrix: slot (r * giant + g) * baby + j holds diagonal g * baby + j of chunk r,
// false where that diagonal is past `dimension` (an absent, all-zero plaintext).
PDB_HD bool pnns_resident(const PnnsShape &s, long long slot, int &d, long long &r) {
    const long long per_result = (long long)s.giant * s.baby;
    r = slot / per_result;
    d = (int)(slot - r * per_result);  // g * baby + j
    return d < s.dimension;
}

// PlaintextMatrix.init(signedValues:reduce:): Modulus.reduce (x mod t in [0, t)), or centeredToRemainder, which
// requires x in [-floor(t / 2), floor((t - 1) / 2)] (`bad` is set otherwise).
PDB_HD uint64_t pnns_signed_value(long long x, uint64_t t, bool reduce, bool &bad) {
    const long long m = (long long)t;
    if (reduce) {
        const long long r = x % m;
        return (uint64_t)(r < 0 ? r + m : r);
    }
    if (x > (m - 1) / 2 || x < -(m / 2)) bad = true;
    return x < 0 ? (uint64_t)(x + m) : (uint64_t)x;
}

// ---- PNNS client ----------------------------------------------------------------------------------------------------
// Array2d.normalizedScaledAndRounded (PrivateNearestNeighborSearch/Util.swift:74-89) in Swift Float arithmetic: every
// operation rounded on its own (no contraction into an FMA, whatever the compiler flags), the squares summed left to
// right, a correctly rounded square root, (value * s) / norm as two roundings, then .toNearestOrAwayFromZero.
#ifdef __CUDA_ARCH__
#define PNNS_FMUL(a, b) __fmul_rn(a, b)
#define PNNS_FADD(a, b) __fadd_rn(a, b)
#define PNNS_FDIV(a, b) __fdiv_rn(a, b)
#define PNNS_FSQRT(a) __fsqrt_rn(a)
#else
// the host build that replays these helpers compiles with -ffp-contract=off; a volatile keeps each step rounded anyway
PDB_HD float pnns_round_step(float x) {
    volatile float v = x;
    return v;
}
#define PNNS_FMUL(a, b) pnns_round_step((a) * (b))
#define PNNS_FADD(a, b) pnns_round_step((a) + (b))
#define PNNS_FDIV(a, b) pnns_round_step((a) / (b))
#define PNNS_FSQRT(a) sqrtf(a)
#endif

// row.map { $0 * $0 }.reduce(0, +).squareRoot(): the sum is sequential on purpose -- a reordered sum changes the norm
PDB_HD float pnns_row_norm(const float *row, long long cols) {
    float sum = 0.0f;
    for (long long k = 0; k < cols; ++k) sum = PNNS_FADD(sum, PNNS_FMUL(row[k], row[k]));
    return PNNS_FSQRT(sum);
}

// V((value * scalingFactor / norm).rounded()) with V = Int64; 0 for a zero norm.  `bad` is set where Swift traps: a
// non-finite input (its row's values are NaN) or a rounded value outside Int64.
PDB_HD long long pnns_scaled_value(float value, float scale, float norm, bool &bad) {
    if (!isfinite(value)) {
        bad = true;
        return 0;
    }
    if (norm == 0.0f) return 0;
    const float r = roundf(PNNS_FDIV(PNNS_FMUL(value, scale), norm));
    if (!(r >= -9223372036854775808.0f && r < 9223372036854775808.0f)) {  // also NaN
        bad = true;
        return 0;
    }
    return (long long)r;
}

PDB_HD long long pnns_next_pow2(long long v) {
    long long p = 1;
    while (p < v) p <<= 1;
    return p;
}

// PlaintextMatrix.denseRowPlaintexts (PlaintextMatrix.swift:341-413) for `rows` rows of `cols` values: SIMD slot `slot`
// (0 .. N) of plaintext `p` -> index of the row-major value it holds, -1 for a zero.  Rows take nextPow2(cols) slots
// each, N / nextPow2(cols) rows per plaintext (the SIMD-row padding of :386-388 never applies, as nextPow2(cols)
// divides N / 2).  The last plaintext's k rows are padded to a power of two within their SIMD row and repeated to
// fill N slots (:396-408): [0, P) repeated when they fit in one SIMD row, else the first SIMD row then the second's
// P slots repeated.  The same formula covers full plaintexts (k = N / nextPow2(cols), P = N / 2).
PDB_HD long long pnns_dense_row_element(long long rows, long long cols, int logn, long long p, long long slot) {
    const long long n = 1ll << logn, half = n >> 1, width = pnns_next_pow2(cols), per = n / width;
    const long long left = rows - p * per, k = left < per ? left : per;
    const long long len = k * width;
    long long at;
    if (len <= half) {
        at = slot % pnns_next_pow2(len);
    } else {
        at = slot < half ? slot : half + (slot - half) % pnns_next_pow2(len - half);
    }
    const long long j = at / width, c = at - j * width;
    return j < k && c < cols ? (p * per + j) * cols + c : -1;
}

// ciphertexts of a .denseRow matrix: ceil(rows / (N / nextPow2(cols)))
PDB_HD long long pnns_dense_row_count(long long rows, long long cols, int logn) {
    const long long per = (1ll << logn) / pnns_next_pow2(cols);
    return (rows + per - 1) / per;
}

// PlaintextMatrix.unpackDenseColumn (PlaintextMatrix.swift:515-556) of a rows x cols .denseColumn matrix: element
// (r, c) of the row-major result is column-major value c * rows + r, which plaintext `p` holds at SIMD slot `slot`.
// With 2 * (N/2 / rows) > 1 columns per plaintext, each SIMD row holds rows * (N/2 / rows) values; otherwise a column
// takes ceil(rows / N) plaintexts.
PDB_HD void pnns_dense_column_slot(long long rows, long long cols, int logn, long long r, long long c, long long &p,
                                   long long &slot) {
    const long long n = 1ll << logn, half = n >> 1;
    const long long m = c * rows + r;
    if (2 * (half / rows) > 1) {
        const long long per_row = rows * (half / rows);
        p = m / (2 * per_row);
        const long long w = m - p * 2 * per_row;
        slot = w < per_row ? w : half + (w - per_row);
    } else {
        const long long per_column = (rows + n - 1) / n;
        p = c * per_column + r / n;
        slot = r % n;
    }
    (void)cols;
}

// plaintexts of a rows x cols .denseColumn matrix (the replies mulTranspose(matrix:) returns)
PDB_HD long long pnns_dense_column_count(long long rows, long long cols, int logn) {
    const long long n = 1ll << logn, half = n >> 1;
    if (2 * (half / rows) > 1) {
        const long long per = 2 * rows * (half / rows);
        return (rows * cols + per - 1) / per;
    }
    return cols * ((rows + n - 1) / n);
}

// Plaintext CRT over t_0 .. t_{k-1} (CrtComposer.compose, CrtComposer.swift:76-97), remainderToCentered over T = prod t_i
// and Float(signed) / (Float(s) * Float(s)) (Client.swift:110-117).  x[i] < t[i]; inv[i] = (T / t_i)^-1 mod t_i,
// punct[i] = T / t_i; T below 2^63 when k > 1 (composeMaxIntermediateValue = 2T), so the modular sum never wraps.
struct PnnsCrt {
    int count;
    uint64_t t[8], inv[8], punct[8];
    uint64_t product;
};
PDB_HD long long pnns_crt_signed(const PnnsCrt &c, const uint64_t *x) {
    uint64_t acc = 0;
    for (int i = 0; i < c.count; ++i) {
        const uint64_t tmp = (uint64_t)((unsigned __int128)x[i] * c.inv[i] % c.t[i]);
        const uint64_t add = tmp * c.punct[i];  // < T
        acc += add;
        if (acc >= c.product) acc -= c.product;
    }
    // UInt64.remainderToCentered (Scalar.swift): x > (T - 1) / 2 ? x - T : x
    return acc > (c.product - 1) / 2 ? (long long)(acc - c.product) : (long long)acc;
}
PDB_HD float pnns_distance(long long v, long long scaling_factor) {
#ifdef __CUDA_ARCH__
    const float s = __ll2float_rn(scaling_factor);
    return __fdiv_rn(__ll2float_rn(v), __fmul_rn(s, s));
#else
    const float s = (float)scaling_factor;
    return PNNS_FDIV((float)v, PNNS_FMUL(s, s));
#endif
}

}  // namespace procdb
}  // namespace hecuda
