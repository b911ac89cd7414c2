// kernels.cuh -- launchers of the sm_90a kernels (all take device pointers and a stream).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <string>

#include "context.hpp"

namespace hecuda {

extern std::atomic<unsigned long long> g_kernel_launches;  // every <<<>>> issued by this library

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
// mac: dig (Eval) x key -> prod[item][2][l+1][N] (Eval)
cudaError_t launch_ks_mac(const Context &ctx, const u64 *dig, const u64 *key, int l, u64 *prod, int64_t items,
                          cudaStream_t stream);
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
cudaError_t launch_plaintext_to_eval(const Context &ctx, const u64 *plain, int l, u64 *out, int64_t count,
                                     cudaStream_t stream);

// ---- the plaintext side of Bfv (plaintext.cu); the context must support SIMD encoding for encode / decode
// encodeSimd (+ convertToEvalFormat when l >= 1): values count x value_count (< t) -> out count x N (Coeff, l = 0) or
// count x l x N (Eval).  decodeSimd / decodeEval: plain count x N (l = 0) or count x l x N -> values count x N.
// scratch: simd_scratch_words per item (stream-ordered, caller-owned).
size_t simd_scratch_words(const Context &ctx, bool encode, int l);
cudaError_t launch_encode_simd(const Context &ctx, const u64 *values, int value_count, int l, u64 *out, u64 *scratch,
                               int64_t count, cudaStream_t stream);
cudaError_t launch_decode_simd(const Context &ctx, const u64 *plain, int l, u64 *values, u64 *scratch, int64_t count,
                               cudaStream_t stream);
// plaintextTranslate: ct, out batch x polys x l x N (Coeff); pt N values (< t) shared by all (broadcast) or batch x N;
// op = HECUDA_PLAINTEXT_ADD / SUB / SUB_FROM; out may equal ct
cudaError_t launch_plaintext_translate(const Context &ctx, const u64 *ct, int polys, int l, const u64 *pt, bool broadcast,
                                       int op, u64 *out, int64_t batch, cudaStream_t stream);

// ---- wire format (codec.cu): PolyRq.serialize / load, PolyRq+Serialize.swift:28-84
struct CodecConsts {
    int rows;
    int width[kMaxRows];                  // serialized bits per coefficient of each row
    long long byte_offset[kMaxRows + 1];  // of each row inside one serialized polynomial
};
bool codec_consts(const Context &ctx, const NttRowMap &map, int skip, CodecConsts &c, std::string &err);
long long serialized_poly_bytes(const CodecConsts &c);
cudaError_t launch_poly_load(const Context &ctx, const CodecConsts &c, int skip, const unsigned char *bytes, u64 *out,
                             int64_t polys, cudaStream_t stream);
cudaError_t launch_poly_serialize(const Context &ctx, const CodecConsts &c, int skip, const u64 *in, unsigned char *bytes,
                                  int64_t polys, cudaStream_t stream);

// uint32 <-> uint64 residues at the boundary of a Bfv<UInt32> context (elementwise.cu); both buffers 16-byte aligned
cudaError_t launch_widen(const u32 *in, u64 *out, int64_t words, cudaStream_t stream);
cudaError_t launch_narrow(const u64 *in, u32 *out, int64_t words, cudaStream_t stream);

// divideAndRoundQLast over polys x l x N -> polys x (l-1) x N
cudaError_t launch_mod_switch(const Context &ctx, const u64 *in, int l, u64 *out, int64_t polys, cudaStream_t stream);

}  // namespace hecuda
