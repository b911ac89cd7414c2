// kernels.cuh -- launchers of the sm_90a kernels (all take device pointers and a stream).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <utility>

#include "context.hpp"
#include "process_db.cuh"

namespace hecuda {

extern std::atomic<unsigned long long> g_kernel_launches;  // every <<<>>> issued by this library

// ---- launching.  Every kernel outside the NTT files (ntt_simple.cu, ntt_fast.cu/.cuh) is launched through `launch`,
// so hecuda_kernel_launch_count counts it.
constexpr int64_t kMaxGridYZ = 65535;  // the largest gridDim.y / gridDim.z

// block size of a kernel with one thread per coefficient of an n-coefficient row: n clamped to 32 .. 256
inline int coeff_threads(int64_t n) { return n >= 256 ? 256 : (n < 32 ? 32 : (int)n); }

// one counted launch: kernel<<<grid, block, smem, stream>>>(args...), then the launch's error
template <typename... KArgs, typename... Args>
cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args &&...args) {
    ++g_kernel_launches;
    kernel<<<grid, block, smem, stream>>>(std::forward<Args>(args)...);
    return cudaGetLastError();
}

// body(first, part) for consecutive parts [first, first + part) of [0, count), part <= limit, until one returns an
// error: a batch that a kernel puts in grid y or z is launched in parts of at most kMaxGridYZ
template <typename Body>
cudaError_t for_each_part(int64_t count, Body &&body, int64_t limit = kMaxGridYZ) {
    for (int64_t first = 0; first < count; first += limit) {
        const cudaError_t e = body(first, std::min(limit, count - first));
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// the modulus of each of a polynomial's rows under `map`, for a kernel's parameter block
struct RowModuli {
    int rows;
    u64 p[kMaxRows];
};
inline RowModuli row_moduli(const Context &ctx, const NttRowMap &map) {
    RowModuli m;
    m.rows = map.rows_per_poly;
    for (int r = 0; r < m.rows; ++r) m.p[r] = ctx.slots[map.slot[r]].dev.p;
    return m;
}

// ---- negacyclic NTT over rows (ntt.cu).  data: rows x N, row r uses slot map.slot[r % map.rows_per_poly].
// Forward: natural order in -> bit-reversed out (PolyRq+Ntt.swift:237-319); inverse is its inverse (:379-483).
// scale_t: fold the BFV `poly * t` step (Bfv+Multiply.swift:40) into the inverse transform's N^-1 scaling.
cudaError_t launch_ntt_forward(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               cudaStream_t stream);
cudaError_t launch_ntt_inverse(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               int scale_mode, cudaStream_t stream);

// implementations behind the dispatcher (ntt_simple.cu)
cudaError_t launch_ntt_forward_simple(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                      cudaStream_t stream);
cudaError_t launch_ntt_inverse_simple(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                      int scale_mode, cudaStream_t stream);

// register-tiled kernels (ntt_fast.cu), N = 2^10 .. 2^15
bool ntt_fast_supported(const Context &ctx);
cudaError_t launch_ntt_forward_fast(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                    cudaStream_t stream);
cudaError_t launch_ntt_inverse_fast(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                    int scale_mode, cudaStream_t stream);
// forward NTT of the lifted operands + tensor product in one kernel (ntt_fast.cu), N = 2^13: lhs / rhs (items x 2 x L x N, Coeff, 16-byte aligned) and their auxiliary rows (launch_lift into
// ext[item][4] with q_rows = false) -> ten[item][3][R][N] (Eval, Montgomery form like launch_tensor)
bool ntt_forward_tensor_supported(const Context &ctx);
cudaError_t launch_ntt_forward_tensor(const Context &ctx, const NttRowMap &map, const u64 *lhs, const u64 *rhs,
                                      const u64 *ext, u64 *ten, int64_t items, cudaStream_t stream);

// ---- BEHZ steps of ct x ct multiply (behz.cu).  reference_base: compute over the reference's [Q, Bsk] (stage-level
// entry points) instead of the [Q, aux] base the fused multiply uses (context.hpp).
// lift: lhs (and rhs, unless null), each `items` x polys_in x L x N (polys_in 1 or 2), in one launch  ->
// ext[item][op][p][R][N] with op 0 for lhs, 1 for rhs; q_rows = false: the L + 1 auxiliary rows only
// (ext[item][op][p][L + 1][N]), for a consumer that reads the Q rows from the input itself
cudaError_t launch_lift(const Context &ctx, const u64 *lhs, const u64 *rhs, int polys_in, u64 *ext, int64_t items,
                        cudaStream_t stream, bool reference_base = false, bool q_rows = true);
// tensor: ext[item][4][R][N] (Eval) -> ten[item][3][R][N]
cudaError_t launch_tensor(const Context &ctx, const u64 *ext, u64 *ten, int64_t items, cudaStream_t stream,
                          bool reference_base = false);
// tensor sum: ext[group][pair][4][R][N] (Eval) -> ten[group][3][R][N]  (Bfv.innerProduct(_:_:), Bfv.swift:315-361)
cudaError_t launch_tensor_sum(const Context &ctx, const u64 *ext, u64 *ten, int64_t pairs, int64_t groups,
                              cudaStream_t stream, bool reference_base = false);
// floor: polys x R x N (Coeff, already scaled by t) -> polys x L x N.  q_scaled: the Q rows are already multiplied
// by (Q/q_i)^-1 (an inverse NTT with kScaleTMontFloor instead of kScaleTMont); only where floor_takes_scaled_q
bool floor_takes_scaled_q(const Context &ctx);
cudaError_t launch_floor(const Context &ctx, const u64 *in, u64 *out, int64_t polys, cudaStream_t stream,
                         bool reference_base = false, bool q_scaled = false);

// ---- key switching and modulus switching (keyswitch.cu)
// One key-switching key per client for a launch that switches several clients' items: item i (counted from item0)
// belongs to client i / items_per_client.  Passed in the kernel's parameter block.
constexpr int kKeyTableSize = 16;
struct KsKeyTable {
    const u64 *key[kKeyTableSize];
    long long items_per_client, item0;
};
// mac: dig (Eval) x key -> prod[item][2][l+1][N] (Eval); keys: per-client keys instead of `key`
cudaError_t launch_ks_mac(const Context &ctx, const u64 *dig, const u64 *key, int l, u64 *prod, int64_t items,
                          cudaStream_t stream, const KsKeyTable *keys = nullptr);
// finish: out[item][c][i] = divround(prod[item][c])[i] (+ base[item][c][i] for the components in base_mask)
cudaError_t launch_ks_finish(const Context &ctx, const u64 *prod, const u64 *base, int64_t base_item_stride, int base_mask,
                             int l, u64 *out, int64_t items, cudaStream_t stream);
// ---- Galois automorphisms (galois.cu): PolyRq.applyGalois in Coeff / Eval format (Galois.swift:115-166)
cudaError_t launch_galois_coeff(const Context &ctx, const NttRowMap &map, unsigned element, const u64 *in,
                                int64_t in_poly_stride, u64 *out, int64_t out_poly_stride, int64_t polys,
                                cudaStream_t stream);
cudaError_t launch_multiply_power_of_x(const Context &ctx, const NttRowMap &map, long long power, const u64 *in, u64 *out,
                                       int64_t polys, cudaStream_t stream);
cudaError_t launch_galois_eval(const Context &ctx, int rows, unsigned element, const u64 *in, u64 *out, int64_t polys,
                               cudaStream_t stream);

// ---- lazy ct x pt inner product and plaintext Eval conversion (innerprod.cu): Bfv.swift:476-505, Plaintext.swift:149-171
cudaError_t launch_inner_product_plain(const Context &ctx, const u64 *cts, int npoly, int l, int64_t terms, const u64 *pts,
                                       const unsigned char *present, u64 *out, int64_t out_count, cudaStream_t stream);
// the same scan for moduli below 2^31 with the plaintext rows stored as uint32 (innerprod.cu)
bool inner_product_plain_small_supported(const Context &ctx, int l);
cudaError_t launch_inner_product_plain_small(const Context &ctx, const u64 *cts, int npoly, int l, int64_t terms, const u32 *pts,
                                             const unsigned char *present, u64 *out, int64_t out_count, cudaStream_t stream);
// The same scans for `clients` 2-poly queries at once: client j's `terms` ciphertexts start at cts + j * client_stride,
// its out_count x 2 x l x N results at out + j * out_client_stride.  The client tiles of a row tile are adjacent
// blocks, so a database row comes from HBM about once per launch; every value is the one the single-client scan
// computes.  One client runs the single-client scan itself.  A MulPir group is kScanClientTiles tiles; the PNNS group
// pipeline passes every rotated-state set of its group (clients x query rows) as a client.
constexpr int kScanClientTile = 4, kScanClientTiles = 4, kScanRowTile = 2;  // clients, tiles per MulPir group, rows
cudaError_t launch_inner_product_plain_clients(const Context &ctx, const u64 *cts, int64_t client_stride, int clients, int l,
                                               int64_t terms, const u64 *pts, const u32 *pts32, const unsigned char *present,
                                               u64 *out, int64_t out_client_stride, int64_t out_count, cudaStream_t stream);
cudaError_t launch_plaintext_to_eval(const Context &ctx, const u64 *plain, int l, u64 *out, int64_t count,
                                     cudaStream_t stream);

#ifdef __CUDACC__
// floor(([Q_l]_t m + tThreshold) / t) for m < t (context.hpp, TranslateConsts): the rounding term of plaintextTranslate,
// shared by the translate kernel (plaintext.cu) and the encryption epilogue (client.cu)
__device__ __forceinline__ u64 translate_adjust(u64 m, const TranslateConsts &c) {
    const u64 quot = mulhi64(m, c.q_mod_t_p);
    u64 r = m * c.q_mod_t - quot * c.t;  // [Q_l]_t m - quot t in [0, 2t)
    u64 fl = quot;
    if (r >= c.t) {
        r -= c.t;
        ++fl;
    }
    return fl + (r + c.t_threshold >= c.t ? 1 : 0);
}
#endif

// ---- the plaintext side of Bfv (plaintext.cu); the context must support SIMD encoding for encode / decode
// encodeSimd (+ convertToEvalFormat when l >= 1): values count x value_count (< t) -> out count x N (Coeff, l = 0) or
// count x l x N (Eval).  decodeSimd / decodeEval: plain count x N (l = 0) or count x l x N -> values count x N.
// scratch: simd_scratch_words per item (stream-ordered, caller-owned).
size_t simd_scratch_words(const Context &ctx, bool encode, int l);
cudaError_t launch_encode_simd(const Context &ctx, const u64 *values, int value_count, int l, u64 *out, u64 *scratch,
                               int64_t count, cudaStream_t stream);
cudaError_t launch_decode_simd(const Context &ctx, const u64 *plain, int l, u64 *values, u64 *scratch, int64_t count,
                               cudaStream_t stream);
// NTT of `rows` rows (rows x N), all mod the modulus of one slot (e.g. ctx.slot_t()); the inverse scales by N^-1 only
cudaError_t ntt_single(const Context &ctx, int slot, bool inverse, const u64 *in, u64 *out, int64_t rows, cudaStream_t s);
// plaintextTranslate: ct, out batch x polys x l x N (Coeff); pt N values (< t) shared by all (broadcast) or batch x N;
// op = HECUDA_PLAINTEXT_ADD / SUB / SUB_FROM; out may equal ct
cudaError_t launch_plaintext_translate(const Context &ctx, const u64 *ct, int polys, int l, const u64 *pt, bool broadcast,
                                       int op, u64 *out, int64_t batch, cudaStream_t stream);

// ---- wire format (codec.cu): PolyRq.serialize / load, PolyRq+Serialize.swift:28-84
struct CodecConsts {
    int rows;
    int width[kMaxRows];                  // serialized bits per coefficient of each row
    long long byte_offset[kMaxRows + 1];  // of each row inside one serialized polynomial
    u64 modulus[kMaxRows];                // of each row (a checked load refuses residues >= it)
};
// field i of one row: the `w` bits at bit i * w of the big-endian stream of the row's `row_bytes` bytes at `src`
HE_HD u64 codec_unpack(const unsigned char *__restrict__ src, long long row_bytes, int w, long long i) {
    const long long bit = i * w;
    const long long first = bit >> 3;
    const int shift = (int)(bit & 7);
    u128 acc = 0;  // 9 bytes cover shift + w <= 7 + 64 bits
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        const long long at = first + k;
        acc = (acc << 8) | (u128)(at < row_bytes ? src[at] : 0);
    }
    const u64 mask = w >= 64 ? ~0ull : ((1ull << w) - 1);
    return (u64)(acc >> (72 - shift - w)) & mask;
}
// the inverse: bits [lo_bit, lo_bit + span) (span <= 64) of the big-endian stream of one row's n coefficients at `src`
// (each shifted right by `skip` and cut to `w` bits), stream bit lo_bit as bit span - 1 of the result
template <typename Word>
HE_HD u64 codec_pack(const Word *__restrict__ src, int n, int w, int skip, long long lo_bit, int span) {
    const u64 mask = w >= 64 ? ~0ull : ((1ull << w) - 1);
    const long long hi_bit = lo_bit + span;
    u64 value = 0;
    for (long long coeff = lo_bit / w; coeff < n && coeff * w < hi_bit; ++coeff) {
        const long long begin = coeff * w, end = begin + w;
        const long long lo = begin > lo_bit ? begin : lo_bit, hi = end < hi_bit ? end : hi_bit;
        const int bits = (int)(hi - lo);
        const u64 v = ((u64)src[coeff] >> skip) & mask;
        const u64 field = (v >> (end - hi)) & (bits >= 64 ? ~0ull : ((1ull << bits) - 1));
        value |= bits >= 64 ? field : field << (hi_bit - hi);
    }
    return value;
}
// Where each polynomial's bytes are.  Default: polynomial p at p * serialized_poly_bytes.  With `tag`: a processed
// database's stream staged from byte `base` of the file, in which plaintext `first` + p has `frame` bytes of framing at
// tag[first + p] and, unless it is nil, its rows right after them; tag[first + p + 1] is where the next one starts.
// A PIR file (IndexPirProtocol.swift:336-378) frames each plaintext with its tag byte (frame 1: 1 present, 0 nil); a
// PNNS file (SerializedProcessedDatabase) with its protobuf keys and lengths, the same bytes for every plaintext of a
// matrix (a load, which walked them on the host, passes the rows' own offsets with frame 0).  A load then writes
// present[p], writes zero rows for a nil plaintext, and atomically lowers *bad to (first + p) * rows + row where a
// residue is >= its modulus; a serialization writes the framing too (frame_bytes, or a 0 tag for a nil plaintext).
// With `slot`, plaintext first + p is resident polynomial slot[first + p] of the rows passed, instead of polynomial p.
// Protobuf messages read in place (pir_proto.hpp) pass each polynomial's own offset in `tag` with frame 0, and for seeded
// ciphertexts each 32-byte seed's offset in `seed` (drbg.cu).
constexpr int kMaxFrame = 24;  // two keys and two 10-byte varints at most
struct PolyLayout {
    const long long *tag = nullptr;
    long long base = 0, first = 0;
    unsigned char *present = nullptr;
    unsigned long long *bad = nullptr;
    const long long *slot = nullptr;
    const long long *seed = nullptr;
    int frame = 1;
    unsigned char frame_bytes[kMaxFrame] = {1};
};
// offset from `base` of the rows of plaintext p of a tagged stream (tag[] as in PolyLayout), or -1 for a nil plaintext
HE_HD long long tagged_rows_offset(const long long *tag, long long base, long long p, int frame = 1) {
    return tag[p + 1] - tag[p] > frame ? tag[p] + frame - base : -1;
}
bool codec_consts(const Context &ctx, const NttRowMap &map, int skip, CodecConsts &c, std::string &err);
long long serialized_poly_bytes(const CodecConsts &c);
// bytes -> rows of `Word` (uint64, or uint32 when every modulus is below 2^32)
template <typename Word>
cudaError_t launch_poly_load(const Context &ctx, const CodecConsts &c, int skip, const unsigned char *bytes, Word *out,
                             int64_t polys, cudaStream_t stream, const PolyLayout &layout = PolyLayout{});
template <typename Word>
cudaError_t launch_poly_serialize(const Context &ctx, const CodecConsts &c, int skip, const Word *in, unsigned char *bytes,
                                  int64_t polys, cudaStream_t stream, const PolyLayout &layout = PolyLayout{});

// uint32 <-> uint64 residues at the boundary of a Bfv<UInt32> context (elementwise.cu); both buffers 16-byte aligned
cudaError_t launch_widen(const u32 *in, u64 *out, int64_t words, cudaStream_t stream);
cudaError_t launch_narrow(const u64 *in, u32 *out, int64_t words, cudaStream_t stream);

// ---- the server's data into plaintexts (process_db.cu; index maps in process_db.cuh)
// The device staging budget of the database pipelines: 64 MB per slab
constexpr int64_t kSlabBytes = (int64_t)64 << 20;
// Plaintexts per slab when a database is packed and converted to Eval piecewise: <= 64 MB of coefficients
inline int64_t coefficient_slab(const Context &ctx) {
    const int64_t per = kSlabBytes / (int64_t)(sizeof(u64) * ctx.n);
    return per > 1 ? per : 1;
}
// MulPirServer.process: plaintexts first .. first + items of the database `s` (entries / offsets on the device) ->
// out items x N coefficients (< t), present[items] (0 = nil plaintext)
cudaError_t launch_pir_pack(const procdb::PirShape &s, int n, int64_t first, int64_t items, u64 *out,
                            unsigned char *present, cudaStream_t stream);
// PlaintextMatrix(signedValues:) .diagonal packing + encodeSimd: plaintexts first .. first + items (diagonalPlaintexts'
// order, or hecuda_pnns_matrix's slot order when `resident`) of the row-major matrix `values` (on the device) ->
// out items x N (Coeff, < t).  A value outside the centered range without `reduce` sets *bad.  Needs ctx.simd.
cudaError_t launch_pnns_diagonal(const Context &ctx, const procdb::PnnsShape &s, const int64_t *values, bool reduce,
                                 bool resident, int64_t first, int64_t items, u64 *out, int *bad, cudaStream_t stream);

// Array2d.normalizedScaledAndRounded (pnns_client.cu): vectors rows x cols floats (on the device) -> norms[rows] and
// values rows x cols Int64 (0 for a zero-norm row); a non-finite input or a value outside Int64 sets *bad
cudaError_t launch_pnns_normalize(const float *vectors, int64_t rows, int64_t cols, int64_t scaling_factor, float *norms,
                                  int64_t *values, int *bad, cudaStream_t stream);

// divideAndRoundQLast over polys x l x N -> polys x (l-1) x N
cudaError_t launch_mod_switch(const Context &ctx, const u64 *in, int l, u64 *out, int64_t polys, cudaStream_t stream);

}  // namespace hecuda
