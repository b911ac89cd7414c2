// codec.cu -- the reference's wire format for RNS polynomials on the device (SURVEY.md 8f rank 4).
//
//   PolyRq.serialize(skipLSBs:) / load(from:skipLSBs:)         PolyRq/PolyRq+Serialize.swift:28-84
//   CoefficientPacking.coefficientsToBytes / bytesToCoefficients CoefficientPacking.swift:59-217
//
// Row i of a polynomial is a big-endian bit stream of N fields of ceil(log2 q_i) - skipLSBs bits, padded with zero
// bits to a whole byte; the rows follow each other.  Unpacking on the device lets query ciphertexts cross PCIe at
// ceil(log2 q) bits per coefficient instead of 64, and responses leave the same way.
#include <algorithm>
#include <cstdint>

#include "kernels.cuh"
#include "modarith.cuh"

namespace hecuda {


// offset of polynomial `poly`'s rows in `bytes` under `at` (-1: a nil plaintext)
__device__ __forceinline__ long long poly_bytes_offset(const CodecConsts &c, const PolyLayout &at, int64_t poly) {
    return at.tag ? tagged_rows_offset(at.tag + at.first, at.base, poly, at.frame) : poly * c.byte_offset[c.rows];
}

// the resident polynomial that plaintext `poly` of the layout is
__device__ __forceinline__ int64_t resident_poly(const PolyLayout &at, int64_t poly) {
    return at.slot ? at.slot[at.first + poly] : poly;
}

// bytes -> coefficients: one thread per coefficient
template <typename Word>
__global__ void __launch_bounds__(256) poly_load_kernel(const unsigned char *__restrict__ bytes, Word *__restrict__ out,
                                                       const __grid_constant__ CodecConsts c, int n, int skip,
                                                       const __grid_constant__ PolyLayout at) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int row = blockIdx.y;
    const int64_t poly = blockIdx.z;
    const long long offset = poly_bytes_offset(c, at, poly);
    if (at.present && row == 0 && i == 0) at.present[poly] = offset >= 0;
    Word *dst = out + (resident_poly(at, poly) * c.rows + row) * n + i;
    if (offset < 0) {
        *dst = 0;
        return;
    }
    const long long row_bytes = c.byte_offset[row + 1] - c.byte_offset[row];
    const u64 v = codec_unpack(bytes + offset + c.byte_offset[row], row_bytes, c.width[row], i) << skip;
    if (at.bad && v >= c.modulus[row]) atomicMin(at.bad, (unsigned long long)(at.first + poly) * c.rows + row);
    *dst = (Word)v;
}

// the framing of a tagged stream's plaintext (a nil plaintext's: its 0 tag), written by the first thread of its first row
__device__ __forceinline__ void write_tag(unsigned char *bytes, const PolyLayout &at, int64_t poly, long long offset, long long j) {
    if (!at.tag || blockIdx.y != 0 || j != 0) return;
    unsigned char *dst = bytes + at.tag[at.first + poly] - at.base;
    if (offset < 0) {
        *dst = 0;
        return;
    }
    for (int k = 0; k < at.frame; ++k) dst[k] = at.frame_bytes[k];
}

// coefficients -> bytes: one thread per output byte
template <typename Word>
__global__ void __launch_bounds__(256) poly_serialize_kernel(const Word *__restrict__ in, unsigned char *__restrict__ bytes,
                                                            const __grid_constant__ CodecConsts c, int n, int skip,
                                                            const __grid_constant__ PolyLayout at) {
    const int row = blockIdx.y;
    const int64_t poly = blockIdx.z;
    const long long row_bytes = c.byte_offset[row + 1] - c.byte_offset[row];
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= row_bytes) return;
    const long long offset = poly_bytes_offset(c, at, poly);
    write_tag(bytes, at, poly, offset, j);
    if (offset < 0) return;
    const u64 value = codec_pack(in + (resident_poly(at, poly) * c.rows + row) * n, n, c.width[row], skip, 8 * j, 8);
    bytes[offset + c.byte_offset[row] + j] = (unsigned char)value;
}

static int ceil_log2_u64(u64 q) {  // T.ceilLog2
    int bits = 0;
    while (bits < 64 && (q - 1) >> bits) ++bits;
    return q <= 1 ? 0 : bits;
}

bool codec_consts(const Context &ctx, const NttRowMap &map, int skip, CodecConsts &c, std::string &err) {
    c.rows = map.rows_per_poly;
    c.byte_offset[0] = 0;
    for (int r = 0; r < c.rows; ++r) {
        const int bits = ceil_log2_u64(ctx.slots[map.slot[r]].dev.p);
        if (!(bits > 0 && bits > skip && skip >= 0)) {  // CoefficientPacking.validate (CoefficientPacking.swift:26-30)
            err = "invalidCoefficientPacking(bitsPerCoeff: " + std::to_string(bits) + ", skipLSBs: " + std::to_string(skip) + ")";
            return false;
        }
        c.width[r] = bits - skip;
        c.byte_offset[r + 1] = c.byte_offset[r] + ((long long)ctx.n * c.width[r] + 7) / 8;
        c.modulus[r] = ctx.slots[map.slot[r]].dev.p;
    }
    return true;
}

long long serialized_poly_bytes(const CodecConsts &c) { return c.byte_offset[c.rows]; }

// `at` for the polynomials from `done` on: a tagged layout moves its first plaintext, the default one its pointers
// (with slots, the rows' pointer stays where it is: the slots are indices into it)
PolyLayout layout_from(const PolyLayout &at, int64_t done) {
    PolyLayout part = at;
    part.first += done;
    if (part.present) part.present += done;
    return part;
}

template <typename Word>
cudaError_t launch_poly_load(const Context &ctx, const CodecConsts &c, int skip, const unsigned char *bytes, Word *out,
                             int64_t polys, cudaStream_t stream, const PolyLayout &layout) {
    const int threads = coeff_threads(ctx.n);
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), (unsigned)c.rows, (unsigned)chunk);
        return launch(poly_load_kernel<Word>, grid, threads, 0, stream, layout.tag ? bytes : bytes + done * c.byte_offset[c.rows],
                      out + (layout.slot ? 0 : done * c.rows * ctx.n), c, (int)ctx.n, skip, layout_from(layout, done));
    });
}

// coefficients -> bytes, 8 output bytes per thread (rows whose byte count and offset are multiples of 8: N >= 64).
// A tagged stream's rows start right after their framing (a tag byte, or a PNNS file's protobuf keys and lengths), so
// mostly off an 8-byte boundary: the 8 bytes then go out in the widest stores that the rows' alignment allows, the same
// for every thread of the block.
template <typename Word>
__global__ void __launch_bounds__(256) poly_serialize_words_kernel(const Word *__restrict__ in, unsigned char *__restrict__ bytes,
                                                                  const __grid_constant__ CodecConsts c, int n, int skip,
                                                                  const __grid_constant__ PolyLayout at) {
    const int row = blockIdx.y;
    const int64_t poly = blockIdx.z;
    const long long row_words = (c.byte_offset[row + 1] - c.byte_offset[row]) >> 3;
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= row_words) return;
    const long long offset = poly_bytes_offset(c, at, poly);
    write_tag(bytes, at, poly, offset, j);
    if (offset < 0) return;
    // big-endian bit stream: stream bit 64 j is the MSB of the value
    const u64 value = codec_pack(in + (resident_poly(at, poly) * c.rows + row) * n, n, c.width[row], skip, 64 * j, 64);
    // store most significant byte first
    const u64 swapped = __byte_perm((unsigned)(value >> 32), 0, 0x0123) | ((u64)__byte_perm((unsigned)value, 0, 0x0123) << 32);
    unsigned char *dst = bytes + offset + c.byte_offset[row] + 8 * j;
    switch (reinterpret_cast<uintptr_t>(dst) & 7) {
    case 0:
        *reinterpret_cast<u64 *>(dst) = swapped;
        break;
    case 4:
        for (int k = 0; k < 2; ++k) reinterpret_cast<unsigned *>(dst)[k] = (unsigned)(swapped >> (32 * k));
        break;
    case 2:
    case 6:
        for (int k = 0; k < 4; ++k) reinterpret_cast<unsigned short *>(dst)[k] = (unsigned short)(swapped >> (16 * k));
        break;
    default:
        for (int k = 0; k < 8; ++k) dst[k] = (unsigned char)(swapped >> (8 * k));
    }
}

template <typename Word>
cudaError_t launch_poly_serialize(const Context &ctx, const CodecConsts &c, int skip, const Word *in, unsigned char *bytes,
                                  int64_t polys, cudaStream_t stream, const PolyLayout &layout) {
    long long widest = 0;
    // a tagged stream's rows are at least byte aligned; a plain one's must sit on 8-byte boundaries
    bool words = layout.tag || ((reinterpret_cast<uintptr_t>(bytes) & 7) == 0 && (c.byte_offset[c.rows] & 7) == 0);
    for (int r = 0; r < c.rows; ++r) {
        widest = std::max(widest, c.byte_offset[r + 1] - c.byte_offset[r]);
        words = words && (c.byte_offset[r] & 7) == 0 && (c.byte_offset[r + 1] & 7) == 0;
    }
    return for_each_part(polys, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)(((words ? widest / 8 : widest) + 255) / 256), (unsigned)c.rows, (unsigned)chunk);
        return launch(words ? poly_serialize_words_kernel<Word> : poly_serialize_kernel<Word>, grid, 256, 0, stream,
                      in + (layout.slot ? 0 : done * c.rows * ctx.n), layout.tag ? bytes : bytes + done * c.byte_offset[c.rows], c, (int)ctx.n,
                      skip, layout_from(layout, done));
    });
}

template cudaError_t launch_poly_load<u64>(const Context &, const CodecConsts &, int, const unsigned char *, u64 *, int64_t,
                                           cudaStream_t, const PolyLayout &);
template cudaError_t launch_poly_load<u32>(const Context &, const CodecConsts &, int, const unsigned char *, u32 *, int64_t,
                                           cudaStream_t, const PolyLayout &);
template cudaError_t launch_poly_serialize<u64>(const Context &, const CodecConsts &, int, const u64 *, unsigned char *,
                                                int64_t, cudaStream_t, const PolyLayout &);
template cudaError_t launch_poly_serialize<u32>(const Context &, const CodecConsts &, int, const u32 *, unsigned char *,
                                                int64_t, cudaStream_t, const PolyLayout &);

}  // namespace hecuda

// ------------------------------------------------------------------------------------------------ C ABI
#include "capi_internal.hpp"

using namespace hecuda;
using namespace hecuda::api;

namespace {

int32_t codec_setup(const hecuda_context *h, int32_t base, int32_t rows, int32_t skip, const void *a, const void *b,
                    int64_t polys, CodecConsts &c) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (polys < 0 || (polys && (!a || !b))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    NttRowMap map;
    std::string err;
    if (!make_map(*h->ctx, base, rows, map, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    if (!codec_consts(*h->ctx, map, skip, c, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_poly_serialized_byte_count(const hecuda_context *h, int32_t base, int32_t rows, int32_t skip_lsbs,
                                          uint64_t *bytes) {
    CodecConsts c;
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    int32_t rc = codec_setup(h, base, rows, skip_lsbs, nullptr, nullptr, 0, c);
    if (rc) return rc;
    *bytes = (uint64_t)serialized_poly_bytes(c);
    return HECUDA_OK;
}

int32_t hecuda_poly_load_device(const hecuda_context *h, int32_t base, const uint8_t *serialized, int32_t skip_lsbs,
                                uint64_t *out, int32_t rows, int64_t polys, void *stream) {
    CodecConsts c;
    int32_t rc = codec_setup(h, base, rows, skip_lsbs, serialized, out, polys, c);
    if (rc || polys == 0) return rc;
    cudaError_t e = launch_poly_load(*h->ctx, c, skip_lsbs, serialized, (u64 *)out, polys, (cudaStream_t)stream);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "poly_load");
}

int32_t hecuda_poly_serialize_device(const hecuda_context *h, int32_t base, const uint64_t *in, int32_t skip_lsbs,
                                     uint8_t *serialized, int32_t rows, int64_t polys, void *stream) {
    CodecConsts c;
    int32_t rc = codec_setup(h, base, rows, skip_lsbs, in, serialized, polys, c);
    if (rc || polys == 0) return rc;
    cudaError_t e = launch_poly_serialize(*h->ctx, c, skip_lsbs, (const u64 *)in, serialized, polys, (cudaStream_t)stream);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "poly_serialize");
}

int32_t hecuda_poly_load(const hecuda_context *h, int32_t base, const uint8_t *serialized, int32_t skip_lsbs, uint64_t *out,
                         int32_t rows, int64_t polys) {
    CodecConsts c;
    int32_t rc = codec_setup(h, base, rows, skip_lsbs, serialized, out, polys, c);
    if (rc || polys == 0) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const size_t in_bytes = (size_t)serialized_poly_bytes(c) * polys, out_words = (size_t)rows * h->ctx->n * polys;
    cudaStream_t s = g.w->stream;
    unsigned char *d_in = nullptr;
    u64 *d_out = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_in, in_bytes, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_out, out_words * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, serialized, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = launch_poly_load(*h->ctx, c, skip_lsbs, d_in, d_out, polys, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, out_words * sizeof(u64), cudaMemcpyDeviceToHost, s);
    if (d_in) cudaFreeAsync(d_in, s);
    if (d_out) cudaFreeAsync(d_out, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "poly_load");
}

int32_t hecuda_poly_serialize(const hecuda_context *h, int32_t base, const uint64_t *in, int32_t skip_lsbs,
                              uint8_t *serialized, int32_t rows, int64_t polys) {
    CodecConsts c;
    int32_t rc = codec_setup(h, base, rows, skip_lsbs, in, serialized, polys, c);
    if (rc || polys == 0) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const size_t out_bytes = (size_t)serialized_poly_bytes(c) * polys, in_words = (size_t)rows * h->ctx->n * polys;
    cudaStream_t s = g.w->stream;
    unsigned char *d_out = nullptr;
    u64 *d_in = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&d_in, in_words * sizeof(u64), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void **)&d_out, out_bytes, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, in, in_words * sizeof(u64), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = launch_poly_serialize(*h->ctx, c, skip_lsbs, d_in, d_out, polys, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(serialized, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
    if (d_in) cudaFreeAsync(d_in, s);
    if (d_out) cudaFreeAsync(d_out, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = e2;
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "poly_serialize");
}

}  // extern "C"
