/*
 * hecuda.h -- C ABI of the H100-native RNS-BFV polynomial-arithmetic engine (libhecuda.so).
 *
 * This is the drop-in boundary for the hot path of apple/swift-homomorphic-encryption: a SwiftPM C target placed
 * beside Sources/CUtil (the reference's only C target, Package.swift:100-105, Sources/CUtil/zeroize.h:20-26) exposes
 * this header; an in-package overlay of Bfv<UInt64> calls it from the HeScheme entry points listed below
 * (INTEGRATION.md shows the Swift side).  Every entry point cites the reference interface it replaces, with paths
 * relative to the reference checkout.
 *
 * Conventions
 *   - All polynomial data is unsigned 64-bit, little-endian, laid out exactly like the reference's
 *     Array2d<UInt64> (Sources/HomomorphicEncryption/Array2d.swift:19-29,115-123): a polynomial is `rows x N`
 *     row-major, row i holding the residues mod the i-th modulus; a ciphertext is its polynomials back to back
 *     (Ciphertext.polys, Ciphertext.swift:18-28); a batch is ciphertexts back to back.
 *     Coeff format = coefficient order, Eval format = the reference's bit-reversed NTT order.
 *   - Every value read or written is the canonical residue in [0, q_i) (PolyRq.swift:36,85-95).
 *   - Pointers are borrowed for the duration of the call only.  Functions without a `_device` suffix take HOST
 *     pointers and return when the outputs are complete; `_device` variants take device pointers on the current
 *     device and enqueue on `stream` (a cudaStream_t passed as void*; NULL = the legacy default stream) without
 *     synchronizing.
 *   - Return value: HECUDA_OK or a negative status; hecuda_last_error() gives the message for the calling thread
 *     (maps onto the reference's `throws HeError`, Sources/HomomorphicEncryption/Error.swift:17-54).
 *   - All entry points are thread-safe (HeScheme statics are called from concurrent TaskGroup tasks,
 *     Sources/HomomorphicEncryption/Util.swift:141-173); contexts and keys are immutable after creation.
 */
#ifndef HECUDA_H
#define HECUDA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hecuda_context hecuda_context; /* Context<Bfv<UInt64>>, Context.swift:19 */
typedef struct hecuda_comm hecuda_comm;       /* NCCL communicator of the key broadcast (no reference counterpart) */
typedef struct hecuda_evk hecuda_evk;         /* EvaluationKey<Bfv<UInt64>>, Keys.swift:66-99,222 */
typedef struct hecuda_pnns_matrix hecuda_pnns_matrix;   /* PlaintextMatrix<Bfv<UInt64>, Eval>, .diagonal packing */
typedef struct hecuda_pir_database hecuda_pir_database; /* ProcessedDatabase<Bfv<UInt64>>, IndexPir/IndexPirDatabase.swift */

enum {
    HECUDA_OK = 0,
    HECUDA_ERR_INVALID_ARGUMENT = -1,  /* HeError.invalidCiphertext / invalidPolyContext / invalidDegree ... */
    HECUDA_ERR_UNSUPPORTED = -2,       /* HeError.unsupportedHeOperation */
    HECUDA_ERR_CUDA = -3,              /* device failure (no reference equivalent) */
    HECUDA_ERR_NO_DEVICE = -4,         /* the library never falls back to a CPU path */
    HECUDA_ERR_MISSING_KEY = -5        /* HeError.missingRelinearizationKey / missingGaloisKey */
};

/* Which RNS base the rows of a polynomial are under (selects the NTT tables per row). */
enum {
    HECUDA_BASE_Q = 0,         /* ciphertext context q_0..q_{rows-1}            (Context.swift:102-112) */
    HECUDA_BASE_Q_BSK = 1,     /* [q_0..q_{L-1}, Bsk], rows = 2L+1               (RnsTool.swift:228-233) */
    HECUDA_BASE_KEYSWITCH = 2, /* q_0..q_{rows-2}, q_ks                          (Context.swift:114-127) */
    HECUDA_BASE_Q_AUX = 3      /* [q_0..q_{L-1}, aux], rows = 2L+1: the base hecuda_bfv_multiply computes in.  Its
                                  auxiliary primes are below 2^55 when BEHZ's exactness conditions allow (they do for
                                  every predefined parameter set), else they are Bsk; the product does not depend on the
                                  choice (csrc/context.cu).  HECUDA_AUX_BASE=reference in the environment forces Bsk. */
};

int32_t hecuda_version(void);
const char *hecuda_last_error(void);
int32_t hecuda_device_count(int32_t *count);
int32_t hecuda_set_device(int32_t device); /* one process (or thread) per GPU; contexts belong to a device */

/* Host-side NUMA placement for the GPU `device`: restricts the calling thread (and threads it creates afterwards) to
 * the CPUs local to the GPU's PCIe root and prefers that NUMA node for page allocations, so that staging buffers
 * allocated afterwards with hecuda_host_alloc sit next to the GPU.  One process per GPU calls it once after
 * hecuda_set_device.  numa_node = -1 when the platform does not report one (then nothing is changed).  The reference
 * has no counterpart (it never leaves the host); a Swift host calls this beside its first use of the context. */
int32_t hecuda_bind_host_to_device(int32_t device, int32_t *numa_node, int32_t *cpu_count);
/* Pinned host buffers for the host-pointer entry points (pageable memory works too, but cannot overlap copies). */
int32_t hecuda_host_alloc(void **ptr, uint64_t bytes);
int32_t hecuda_host_free(void *ptr);
int32_t hecuda_host_register(void *ptr, uint64_t bytes); /* pin an existing allocation, e.g. a Swift array buffer */
int32_t hecuda_host_unregister(void *ptr);

/* Context<Bfv<UInt64>>.init(encryptionParameters:)  -- Context.swift:94-143.
 * coefficient_moduli = q_0..q_{L-1}, q_ks (the last one is reserved for key switching, Context.swift:102-107);
 * all must be NTT-friendly primes < 2^62.  Builds NTT tables (PolyRq+Ntt.swift:118-169), the BEHZ base and
 * constants (RnsTool.swift:30-33,132-251) and key-/mod-switch constants (PolyContext.swift:108-111). */
int32_t hecuda_context_create(int64_t poly_degree, const uint64_t *coefficient_moduli, int32_t moduli_count,
                              uint64_t plaintext_modulus, hecuda_context **out);
/* Context<Bfv<UInt32>>: the reference's 32-bit scalar type (HeScheme.swift, ModularArithmetic/Scalar.swift:498-511) --
 * moduli below 2^30, m~ = 2^16, rnsCorrectionFactor 2^30 - 20405, 29-bit Bsk primes.  Buffers of the hecuda_u32_* entry
 * points are uint32_t in the same layouts as their uint64_t counterparts; residues cross PCIe as 4 bytes and the NTT
 * butterflies run in 32-bit arithmetic.  The uint64_t entry points also accept such a context (64-bit storage of the
 * same residues); the application drivers (MulPir / PNNS), the codec and decryption are uint64_t-only. */
int32_t hecuda_context_create_u32(int64_t poly_degree, const uint32_t *coefficient_moduli, int32_t moduli_count,
                                  uint32_t plaintext_modulus, hecuda_context **out);
int32_t hecuda_context_word_bits(const hecuda_context *ctx, int32_t *bits); /* 64 or 32 */
int32_t hecuda_context_destroy(hecuda_context *ctx);
/* Introspection used by the parity tests (the reference exposes the same values as public lets). */
int32_t hecuda_context_ciphertext_moduli_count(const hecuda_context *ctx, int32_t *count);
int32_t hecuda_context_bsk_moduli(const hecuda_context *ctx, uint64_t *out, int32_t capacity, int32_t *count);
/* The L+1 auxiliary primes of HECUDA_BASE_Q_AUX (equal to Bsk when the faster base is not admissible). */
int32_t hecuda_context_aux_moduli(const hecuda_context *ctx, uint64_t *out, int32_t capacity, int32_t *count);
/* rootOfUnityPowers / inverse powers of `modulus` in the reference's bit-reversed order (PolyRq+Ntt.swift:125-137);
 * inverse table is indexed like the forward one (inv[i] = roots[i]^-1). */
int32_t hecuda_context_root_tables(const hecuda_context *ctx, uint64_t modulus, uint64_t *roots, uint64_t *inverse_roots);

/* _RnsTool.liftQToQBsk (RnsTool.swift:324-331) and _RnsTool.floorQBskToQ (RnsTool.swift:453-456) at the top level, on
 * their own: Coeff-format polynomials, host pointers.  lift: poly_count x L x N canonical residues mod q_i ->
 * poly_count x (2L+1) x N over [q_0..q_{L-1}, Bsk]; floor: poly_count x (2L+1) x N (the caller has already multiplied by
 * t, Bfv+Multiply.swift:40) -> poly_count x L x N.  These run over the reference's Bsk whatever base hecuda_bfv_multiply
 * uses internally (HECUDA_BASE_Q_AUX). */
int32_t hecuda_rnstool_lift_q_to_qbsk(const hecuda_context *ctx, const uint64_t *polys, uint64_t *out, int64_t poly_count);
int32_t hecuda_rnstool_floor_qbsk_to_q(const hecuda_context *ctx, const uint64_t *polys, uint64_t *out, int64_t poly_count);

/* PolyRq.forwardNtt() / inverseNtt() -- PolyRq+Ntt.swift:230,541 (PolyContext.forwardNtt(poly:) :209-222,
 * inverseNtt(poly:) :524-533), batched: data = poly_count x row_count x N, in place. */
int32_t hecuda_ntt_forward(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count, int64_t poly_count);
int32_t hecuda_ntt_inverse(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count, int64_t poly_count);
int32_t hecuda_ntt_forward_device(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count,
                                  int64_t poly_count, void *stream);
int32_t hecuda_ntt_inverse_device(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count,
                                  int64_t poly_count, void *stream);
/* PolyContext.forwardNtt(dataPtr:modulus:) -- PolyRq+Ntt.swift:329-347: rows of N residues, all mod `modulus`. */
int32_t hecuda_ntt_forward_rows(const hecuda_context *ctx, uint64_t modulus, uint64_t *data, int64_t row_count);
int32_t hecuda_ntt_inverse_rows(const hecuda_context *ctx, uint64_t modulus, uint64_t *data, int64_t row_count);

/* Bfv.mulAssign(_:_:) -- Bfv/Bfv+Multiply.swift:18-21 (multiplyWithoutScaling :63-85 + dropExtendedBase :31-48).
 * lhs, rhs: batch x 2 x L x N (Coeff, top level, correction factor 1); out: batch x 3 x L x N (Coeff).
 * TOP LEVEL ONLY, by construction: the entry point has no moduli_count argument and always reads L rows per polynomial,
 * so a caller holding ciphertexts below the top level (after modSwitchDown) must not pass them here -- the Swift overlay
 * checks `ciphertext.moduli.count == context.ciphertextContext.moduli.count` and throws
 * HeError.unsupportedHeOperation otherwise (INTEGRATION.md).  Reason: below the top level the reference derives its
 * [Bsk, m~] base by dropping m~ from the top-level one (RnsTool.swift:185-186 with PolyContext.swift:131-141) while
 * smallMontgomeryReduce still assumes it (:340-360); no reference test pins what that computes, so it is not
 * reproduced (DESIGN.md "levels").  MulPir and PNNS multiply at the top level only. */
int32_t hecuda_bfv_multiply(const hecuda_context *ctx, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                            int64_t batch);
int32_t hecuda_bfv_multiply_device(const hecuda_context *ctx, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                   int64_t batch, void *stream);

/* EvaluationKey upload.  relin_key = the _KeySwitchKey of the relinearization key (Keys.swift:66-99, generated by
 * Bfv+Keys.swift:58-103): L ciphertexts x 2 polys x K x N in Eval format, K = L + 1 rows under [q_0..q_{L-1}, q_ks]. */
int32_t hecuda_evk_create(const hecuda_context *ctx, const uint64_t *relin_key, hecuda_evk **out);
int32_t hecuda_evk_destroy(hecuda_evk *evk);
/* NCCL-free plumbing for multi-GPU setup: raw device pointer + size of the key so that torch.distributed /
 * ncclBroadcast can replicate it from rank 0 (SURVEY.md section 8e). */
int32_t hecuda_evk_create_empty(const hecuda_context *ctx, hecuda_evk **out);
int32_t hecuda_evk_device_buffer(hecuda_evk *evk, void **device_ptr, uint64_t *bytes);

/* Multi-GPU setup (SURVEY.md section 8e): ciphertext batches shard over the GPUs with no data-path collective; the only
 * exchange is the evaluation key, broadcast once over NCCL (NVLink / NVSwitch) from the rank that received it from the
 * client.  One process per GPU.  Rank 0 calls hecuda_comm_unique_id and hands the 128 bytes to the other ranks over the
 * host's own channel; every rank then calls hecuda_comm_create (collective), creates its key -- hecuda_evk_create with
 * the key material on the root, hecuda_evk_create_empty elsewhere -- and calls hecuda_evk_broadcast (collective) with
 * the same has_relin flag and Galois element list (the EvaluationKeyConfig, known to every rank, Keys.swift:228-262).
 * NCCL is opened at run time (libnccl.so.2, or $HECUDA_NCCL_LIBRARY); without it these return HECUDA_ERR_UNSUPPORTED. */
#define HECUDA_COMM_UNIQUE_ID_BYTES 128
int32_t hecuda_comm_unique_id(uint8_t *id /* HECUDA_COMM_UNIQUE_ID_BYTES */);
int32_t hecuda_comm_create(const uint8_t *id, int32_t rank, int32_t world_size, hecuda_comm **out);
int32_t hecuda_comm_destroy(hecuda_comm *comm);
int32_t hecuda_evk_broadcast(hecuda_evk *evk, hecuda_comm *comm, int32_t root, int32_t has_relin, const uint32_t *elements,
                             int32_t element_count);

/* Bfv.relinearize(_:using:) -- Bfv/Bfv.swift:201-219 (key switch: Bfv+Keys.swift:123-208).
 * ct3: batch x 3 x l x N (Coeff), l = moduli_count in [1, L]; out: batch x 2 x l x N (Coeff). */
int32_t hecuda_bfv_relinearize(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ct3,
                               int32_t moduli_count, uint64_t *out, int64_t batch);
int32_t hecuda_bfv_relinearize_device(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ct3,
                                      int32_t moduli_count, uint64_t *out, int64_t batch, void *stream);

/* Bfv.relinearize followed by Bfv.modSwitchDown in one pass (host pointers): ct3: batch x 3 x l x N -> out: batch x 2 x
 * (l-1) x N; the relinearized ciphertext stays on the device.  Same residues as the two separate calls. */
int32_t hecuda_bfv_relinearize_mod_switch_down(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ct3,
                                               int32_t moduli_count, uint64_t *out, int64_t batch);

/* Bfv.mulAssign, Bfv.relinearize and (mod_switch != 0) Bfv.modSwitchDown in one pass over a batch -- the sequence the
 * reference's callers run back to back (RlweBenchmark.swift:387-493; PirUtil.swift:447-480).  The three-polynomial
 * product never leaves the device: lhs, rhs: batch x 2 x L x N (Coeff, top level); out: batch x 2 x L x N, or
 * batch x 2 x (L-1) x N with the modulus switch.  Same residues as the three separate calls. */
int32_t hecuda_bfv_multiply_relinearize(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *lhs,
                                        const uint64_t *rhs, int32_t mod_switch, uint64_t *out, int64_t batch);
int32_t hecuda_bfv_multiply_relinearize_device(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *lhs,
                                               const uint64_t *rhs, int32_t mod_switch, uint64_t *out, int64_t batch,
                                               void *stream);

/* Bfv.modSwitchDown(_:) -- Bfv/Bfv.swift:163-171 (PolyRq.divideAndRoundQLast, PolyRq.swift:365-393).
 * ct: batch x poly_count x l x N (Coeff), l = moduli_count in [2, L]; out: batch x poly_count x (l-1) x N. */
int32_t hecuda_bfv_mod_switch_down(const hecuda_context *ctx, const uint64_t *ct, int32_t poly_count,
                                   int32_t moduli_count, uint64_t *out, int64_t batch);
int32_t hecuda_bfv_mod_switch_down_device(const hecuda_context *ctx, const uint64_t *ct, int32_t poly_count,
                                          int32_t moduli_count, uint64_t *out, int64_t batch, void *stream);

/* ---- Galois automorphisms (SURVEY.md section 8f, rank 1) ----
 * GaloisKey upload: the _KeySwitchKey for `element` from EvaluationKey.galoisKey.keys (Keys.swift:150-163, generated by
 * Bfv+Keys.swift:42-49), same L x 2 x K x N Eval layout as the relinearization key.  Use hecuda_evk_create_empty for
 * an evaluation key that holds Galois keys only. */
int32_t hecuda_evk_set_galois_key(hecuda_evk *evk, uint32_t element, const uint64_t *key);
/* Device buffer of the key for `element` (allocated if absent), for multi-GPU setups that fill it with a collective
 * the way hecuda_evk_device_buffer does for the relinearization key. */
int32_t hecuda_evk_galois_device_buffer(hecuda_evk *evk, uint32_t element, void **device_ptr, uint64_t *bytes);
/* Bfv.applyGalois(ciphertext:element:using:) -- Bfv/Bfv.swift:174-198 (rotateColumns / swapRows call this with
 * GaloisElement.rotatingColumns / swappingRows, HeScheme.swift:1463-1478).  ct, out: batch x 2 x l x N (Coeff). */
int32_t hecuda_bfv_apply_galois(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ct,
                                int32_t moduli_count, uint32_t element, uint64_t *out, int64_t batch);
int32_t hecuda_bfv_apply_galois_device(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ct,
                                       int32_t moduli_count, uint32_t element, uint64_t *out, int64_t batch, void *stream);
/* PolyRq.applyGalois(element:) in Coeff (eval_format = 0) or Eval (1) format -- PolyRq/Galois.swift:115-141,151-166.
 * in, out: poly_count x row_count x N under `base`; out of place. */
int32_t hecuda_poly_apply_galois(const hecuda_context *ctx, int32_t base, int32_t eval_format, const uint64_t *in,
                                 uint64_t *out, int32_t row_count, int64_t poly_count, uint32_t element);

/* PolyRq<Coeff>.multiplyPowerOfX(_:) -- PolyRq/PolyRq.swift:398-422 (MulPir query expansion, PirUtil.swift:204-241):
 * multiplication by X^power (power may be negative) in Z_q[X]/(X^N + 1); in, out: poly_count x row_count x N. */
int32_t hecuda_poly_multiply_power_of_x(const hecuda_context *ctx, int32_t base, const uint64_t *in, uint64_t *out,
                                        int32_t row_count, int64_t poly_count, int64_t power);

/* ---- lazy ciphertext x plaintext inner product (SURVEY.md section 8f, rank 2) ----
 * Bfv.innerProduct(ciphertexts:plaintexts:) -- Bfv/Bfv.swift:476-505 (lazyMultiply :388-400 over
 * PolyRq.addingLazyProduct, PolyRq.swift:210-225; reduceInPlace/reduceToCiphertext :365-394), batched over
 * `out_count` plaintext rows that share the same `term_count` ciphertexts (the MulPir first-dimension scan,
 * PrivateInformationRetrieval/IndexPir/PirUtil.swift:437-442).  All operands in Eval format.
 *   ciphertexts: term_count x poly_count x l x N       plaintexts: out_count x term_count x l x N
 *   present:     out_count x term_count bytes, 0 = nil plaintext (skipped, Bfv.swift:493); NULL = all present
 *   out:         out_count x poly_count x l x N        out[o] = sum_k ciphertexts[k] * plaintexts[o][k]  (mod q) */
int32_t hecuda_bfv_inner_product_plaintexts(const hecuda_context *ctx, const uint64_t *ciphertexts, int32_t poly_count,
                                            int32_t moduli_count, int64_t term_count, const uint64_t *plaintexts,
                                            const uint8_t *present, uint64_t *out, int64_t out_count);
int32_t hecuda_bfv_inner_product_plaintexts_device(const hecuda_context *ctx, const uint64_t *ciphertexts,
                                                   int32_t poly_count, int32_t moduli_count, int64_t term_count,
                                                   const uint64_t *plaintexts, const uint8_t *present, uint64_t *out,
                                                   int64_t out_count, void *stream);
/* Bfv.innerProduct(_:_:) over ciphertext pairs -- Bfv/Bfv.swift:315-361 (BEHZ multiply with a shared lazy accumulator,
 * one dropExtendedBase for the whole sum), batched over `group_count` independent inner products of `pair_count` pairs:
 * lhs, rhs: group_count x pair_count x 2 x L x N (Coeff, top level); out: group_count x 3 x L x N (Coeff). */
int32_t hecuda_bfv_inner_product(const hecuda_context *ctx, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                 int64_t pair_count, int64_t group_count);
int32_t hecuda_bfv_inner_product_device(const hecuda_context *ctx, const uint64_t *lhs, const uint64_t *rhs, uint64_t *out,
                                        int64_t pair_count, int64_t group_count, void *stream);
/* Plaintext.convertToEvalFormat(moduliCount:) -- Plaintext.swift:149-171 (database preprocessing): `count` coefficient
 * plaintexts of N values < t  ->  count x l x N residues in Eval format. */
int32_t hecuda_plaintext_to_eval(const hecuda_context *ctx, const uint64_t *plain, int32_t moduli_count, uint64_t *out,
                                 int64_t count);
int32_t hecuda_plaintext_to_eval_device(const hecuda_context *ctx, const uint64_t *plain, int32_t moduli_count,
                                        uint64_t *out, int64_t count, void *stream);

/* ---- the plaintext side of Bfv: SIMD batching and ciphertext +- plaintext ----
 * Context.supportsSimdEncoding (Context.swift:63-65): the plaintext modulus t is a prime = 1 mod 2N (isNttModulus,
 * PolyRq+Ntt.swift:24-27).  Such a context also holds t's NTT tables (Context.plaintextContext), so
 * hecuda_ntt_forward_rows / hecuda_ntt_inverse_rows and hecuda_context_root_tables accept `modulus` = t. */
int32_t hecuda_context_supports_simd(const hecuda_context *ctx, int32_t *supported);
/* Context.encode(values:format: .simd) (Encoding.swift:197-235, encodeSimd) and, with moduli_count = l >= 1,
 * Bfv.encode(context:values:format:moduliCount:) (Bfv+Encode.swift:45-50, + Plaintext.convertToEvalFormat).
 * values: count x value_count (value_count <= N, each < t; slots past value_count are zero).  moduli_count 0 -> out
 * count x N Coeff plaintexts; l in [1, L] -> out count x l x N Eval plaintexts.  HECUDA_ERR_UNSUPPORTED without SIMD
 * support (HeError.simdEncodingNotSupported); value_count > N (encodingDataCountExceedsLimit) or, on the host entry
 * point, a value >= t (encodingDataOutOfBounds, Encoding.swift:147-156) -> HECUDA_ERR_INVALID_ARGUMENT.  The _device
 * variant takes values < t as a precondition. */
int32_t hecuda_bfv_encode_simd(const hecuda_context *ctx, const uint64_t *values, int32_t value_count,
                               int32_t moduli_count, uint64_t *out, int64_t count);
int32_t hecuda_bfv_encode_simd_device(const hecuda_context *ctx, const uint64_t *values, int32_t value_count,
                                      int32_t moduli_count, uint64_t *out, int64_t count, void *stream);
/* Context.decode(plaintext:format: .simd) (Encoding.swift:237-245, decodeSimd) and Bfv.decodeEval (Bfv+Encode.swift:76-80,
 * Plaintext.convertToCoeffFormat, Plaintext.swift:176-194).  moduli_count 0: plaintexts count x N Coeff (< t);
 * l in [1, L]: count x l x N Eval plaintexts.  values: count x N slots in [0, t). */
int32_t hecuda_bfv_decode_simd(const hecuda_context *ctx, const uint64_t *plaintexts, int32_t moduli_count,
                               uint64_t *values, int64_t count);
int32_t hecuda_bfv_decode_simd_device(const hecuda_context *ctx, const uint64_t *plaintexts, int32_t moduli_count,
                                      uint64_t *values, int64_t count, void *stream);
/* Bfv.addAssignCoeff / subAssignCoeff (Bfv/Bfv.swift:110-117) and HeScheme.subCoeff (plaintext - ciphertext,
 * HeScheme.swift:1540-1542 = plaintext + -ciphertext): plaintextTranslate (Bfv+Encrypt.swift:75-139) adds or subtracts
 * floor(Q/t) m + floor(([Q]_t m + ceil(t/2)) / t) on poly 0, Q = q_0..q_{l-1}.  ADD and SUB change poly 0 only; SUB_FROM
 * gives [that - c_0] on poly 0 and negates the other polys.  ct, out: batch x poly_count x l x N (Coeff, poly_count 2
 * or 3, l = moduli_count in [1, L], correction factor 1: the caller refuses others, HeError.invalidCorrectionFactor,
 * Bfv+Encrypt.swift:80-82); plaintexts: plaintext_count x N coefficients < t, plaintext_count 1 (shared by every
 * ciphertext) or batch; out may equal ct.  The host entry point refuses a coefficient >= t; the _device variant takes
 * it as a precondition.  Works whether or not the context supports SIMD encoding.  Eval-format ciphertext +- plaintext
 * is not offered: the reference throws unsupportedHeOperation (Bfv.swift:153-160). */
#define HECUDA_PLAINTEXT_ADD 0      /* ct + pt */
#define HECUDA_PLAINTEXT_SUB 1      /* ct - pt */
#define HECUDA_PLAINTEXT_SUB_FROM 2 /* pt - ct */
int32_t hecuda_bfv_plaintext_translate(const hecuda_context *ctx, const uint64_t *ct, int32_t poly_count,
                                       int32_t moduli_count, const uint64_t *plaintexts, int64_t plaintext_count,
                                       int32_t op, uint64_t *out, int64_t batch);
int32_t hecuda_bfv_plaintext_translate_device(const hecuda_context *ctx, const uint64_t *ct, int32_t poly_count,
                                              int32_t moduli_count, const uint64_t *plaintexts, int64_t plaintext_count,
                                              int32_t op, uint64_t *out, int64_t batch, void *stream);

/* ---- MulPir index-PIR server (SURVEY.md section 8f, rank 3) ----
 * Device-resident ProcessedDatabase: `count` optional plaintexts in the order MulPirServer.process emits them
 * (IndexPir/MulPir.swift:433-556: chunk-major, then column-major over the first dimension).  plaintexts is
 * count x L x N in Eval format (eval_format = 1) or count x N coefficient vectors with values < t (eval_format = 0,
 * converted on the device as Plaintext.convertToEvalFormat does, Plaintext.swift:149-171).  present[i] = 0 marks a
 * `nil` plaintext (skipped by the inner product, Bfv.swift:488-494); NULL = all present. */
int32_t hecuda_pir_database_create(const hecuda_context *ctx, const uint64_t *plaintexts, int32_t eval_format,
                                   const uint8_t *present, int64_t count, hecuda_pir_database **out);
int32_t hecuda_pir_database_destroy(hecuda_pir_database *db);
/* The resident rows (for a device-to-device copy between ranks).  When every ciphertext modulus is below 2^31 -- the
 * reference's default PIR parameters -- the rows are kept as uint32 (half the bytes per first-dimension scan) and
 * `bytes` = count * L * N * 4; otherwise uint64 and `bytes` = count * L * N * 8. */
int32_t hecuda_pir_database_device_buffer(hecuda_pir_database *db, void **device_ptr, uint64_t *bytes);

/* PirUtil.expand(ciphertexts:outputCount:using:) -- IndexPir/PirUtil.swift:321-355 (expandCiphertext :249-304,
 * expandCiphertextForOneStep :204-236).  ciphertexts: ciphertext_count x 2 x L x N (Coeff); out: output_count x 2 x L x N,
 * output i encrypting the constant polynomial whose constant is coefficient i of the inputs (x 2^ceilLog2(count)).
 * The Galois keys come from `evk` (hecuda_evk_set_galois_key); the largest configured element <= 2^(logN-logStep+1)+1
 * is applied repeatedly, HECUDA_ERR_MISSING_KEY if none fits (HeError.missingGaloisKey, :216-220). */
int32_t hecuda_mulpir_expand(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ciphertexts,
                             int32_t ciphertext_count, int64_t output_count, uint64_t *out);
int32_t hecuda_mulpir_expand_device(const hecuda_context *ctx, const hecuda_evk *evk, const uint64_t *ciphertexts,
                                    int32_t ciphertext_count, int64_t output_count, uint64_t *out, void *stream);

/* PirUtil.computeResponse(to:using:databases:parameter:context:) -- IndexPir/PirUtil.swift:490-568 with
 * computeResponseForOneChunk (:408-486): expand the query, forward-NTT the first dimension, one ct x pt inner product
 * per database column, one ct x ct inner product + relinearize per further dimension, modSwitchDownToSingle
 * (HeScheme.swift:1481-1485).  dimensions = IndexPirParameter.dimensions, chunk_count =
 * ceil(encodedEntrySize / bytesPerPlaintext) (:507); query: query_ciphertext_count x 2 x L x N (Coeff) holding
 * indices_count queries; database_count is 1 or >= indices_count (PirError.invalidBatchSize otherwise, :498-500).
 * out: indices_count x chunk_count x 2 x 1 x N (Coeff, single modulus q_0) = Response.ciphertexts. */
int32_t hecuda_mulpir_compute_response(const hecuda_context *ctx, const hecuda_evk *evk,
                                       const hecuda_pir_database *const *databases, int32_t database_count,
                                       const int32_t *dimensions, int32_t dimension_count, int32_t chunk_count,
                                       const uint64_t *query, int32_t query_ciphertext_count, int32_t indices_count,
                                       uint64_t *out);
int32_t hecuda_mulpir_compute_response_device(const hecuda_context *ctx, const hecuda_evk *evk,
                                              const hecuda_pir_database *const *databases, int32_t database_count,
                                              const int32_t *dimensions, int32_t dimension_count, int32_t chunk_count,
                                              const uint64_t *query, int32_t query_ciphertext_count,
                                              int32_t indices_count, uint64_t *out, void *stream);

/* The same, bytes in / bytes out: the query ciphertexts as they travel (SerializedCiphertext.seeded: poly0 serialized with
 * skipLSBs 0 over all L rows, plus the 32-byte seed; SerializedCiphertext.swift:41-49,150-154) and the reply ciphertexts as
 * they leave (SerializedCiphertext.full with Bfv.skipLSBsForDecryption, Bfv+Decrypt.swift:51-110: single modulus, poly 0 and
 * poly 1 packed with skip_lsbs_poly0 / skip_lsbs_poly1 dropped bits).  out: indices_count x chunk_count x
 * (byteCount(1 row, skip0) + byteCount(1 row, skip1)) bytes.  Expansion of the seeds, the whole response computation and
 * the packing run on the device; PCIe carries ceil(log2 q) bits per coefficient in and (ceil(log2 q_0) - skip) out. */
int32_t hecuda_mulpir_compute_response_wire(const hecuda_context *ctx, const hecuda_evk *evk,
                                            const hecuda_pir_database *const *databases, int32_t database_count,
                                            const int32_t *dimensions, int32_t dimension_count, int32_t chunk_count,
                                            const uint8_t *query_poly0, const uint8_t *query_seeds,
                                            int32_t query_ciphertext_count, int32_t indices_count, int32_t skip_lsbs_poly0,
                                            int32_t skip_lsbs_poly1, uint8_t *out);

/* ---- PNNS server: encrypted vector x plaintext matrix (SURVEY.md section 8f, rank 3) ----
 * Device-resident PlaintextMatrix in `.diagonal(babyStepGiantStep:)` packing (PrivateNearestNeighborSearch/
 * PlaintextMatrix.swift:417-482): nextPowerOfTwo(column_count) * ceil(row_count / N) plaintexts in the order the
 * reference stores them, either as coefficient vectors (count x N, eval_format = 0; converted on the device like
 * Plaintext.convertToEvalFormat, MatrixMultiplication.swift:206-208) or as count x L x N Eval plaintexts.
 * baby_step / giant_step = BabyStepGiantStep (MatrixMultiplication.swift:26-62). */
int32_t hecuda_pnns_matrix_create(const hecuda_context *ctx, const uint64_t *plaintexts, int32_t eval_format,
                                  int64_t row_count, int64_t column_count, int32_t baby_step, int32_t giant_step,
                                  hecuda_pnns_matrix **out);
int32_t hecuda_pnns_matrix_destroy(hecuda_pnns_matrix *matrix);
int32_t hecuda_pnns_matrix_result_count(const hecuda_pnns_matrix *matrix, int64_t *count); /* ceil(row_count / N) */

/* PlaintextMatrix.mulTranspose(vector:using:) -- MatrixMultiplication.swift:131-226, for `batch` dense-row query
 * ciphertexts (batch x 2 x L x N, Coeff) that share `evk`: babyStep-1 rotateColumns(by: -1), forward NTTs, one
 * ct x pt inner product per (result ciphertext, giant step), rotateColumnsAndSum(by: -babyStep)
 * (_HomomorphicEncryptionExtras/HeScheme.swift:113-134; the Galois keys for both rotations must be in `evk`,
 * HECUDA_ERR_MISSING_KEY otherwise).  mod_switch_to_single = 1 appends Server.computeResponse's
 * modSwitchDownToSingle (Server.swift:79-80).  out: batch x result_count x 2 x (1 or L) x N (Coeff). */
int32_t hecuda_pnns_mul_transpose_vector(const hecuda_context *ctx, const hecuda_evk *evk, const hecuda_pnns_matrix *matrix,
                                         const uint64_t *vectors, int64_t batch, int32_t mod_switch_to_single,
                                         uint64_t *out);
int32_t hecuda_pnns_mul_transpose_vector_device(const hecuda_context *ctx, const hecuda_evk *evk,
                                                const hecuda_pnns_matrix *matrix, const uint64_t *vectors, int64_t batch,
                                                int32_t mod_switch_to_single, uint64_t *out, void *stream);

/* PlaintextMatrix.mulTranspose(matrix:using:) -- MatrixMultiplication.swift:236-298: for every row of the dense-row
 * packed query CiphertextMatrix (ciphertexts: ciphertext_count x 2 x L x N, Coeff) CiphertextMatrix.extractDenseRow
 * (CiphertextMatrix.swift:245-352), the vector product above, then the dense-column packing of the result columns
 * (rotateColumnsAndSum(by: rowCount) + swapRowsAndAdd, _HomomorphicEncryptionExtras/HeScheme.swift:113-151).
 * The caller passes what extractDenseRow derives from the matrix shape for each query row -- the index of the
 * ciphertext holding it, the SIMD-encoded plaintext mask (query_row_count x N coefficients, :300-320), the number of
 * replication rotations (:331-336) -- with column_step = columnCount.nextPowerOfTwo, and the single rotation steps
 * rotateColumnsMultiStep(by: rowCount) resolves to with the configured keys (GaloisElement._planMultiStep,
 * PolyRq/Galois.swift:272-319; the reference iterates that plan in unspecified Dictionary order).  For
 * query_row_count == 1 the row descriptors are ignored (extractDenseRow is the identity).
 * out: *out_count ciphertexts of 2 x (1 or L) x N, the `.denseColumn` CiphertextMatrix; out_capacity in ciphertexts. */
int32_t hecuda_pnns_mul_transpose_matrix(const hecuda_context *ctx, const hecuda_evk *evk, const hecuda_pnns_matrix *matrix,
                                         const uint64_t *ciphertexts, int32_t ciphertext_count, int32_t query_row_count,
                                         const int32_t *row_ciphertext_index, const uint64_t *row_masks,
                                         const int32_t *row_rotate_count, int32_t column_step, const int32_t *pack_rotations,
                                         int32_t pack_rotation_count, int32_t mod_switch_to_single, uint64_t *out,
                                         int64_t out_capacity, int64_t *out_count);

/* ---- coefficient-wise PolyRq arithmetic (SURVEY.md section 8a, row a7) ----
 * PolyRq += / -= (PolyRq/PolyRq.swift:147-174), *= in Eval format (:184-204, Modulus.multiplyMod Modulus.swift:89-94),
 * negation (negateMod, ModularArithmetic/Scalar.swift:167-175) and *= [T] with one reduced scalar per RNS row
 * (:232-245).  In place on lhs / data: poly_count x row_count x N under `base`; results canonical in [0, q_i).
 * Ciphertext += Ciphertext, Ciphertext -= Ciphertext, Ciphertext *= Plaintext (Eval) are these on the polys. */
int32_t hecuda_poly_add(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t row_count,
                        int64_t poly_count);
int32_t hecuda_poly_sub(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t row_count,
                        int64_t poly_count);
int32_t hecuda_poly_mul(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs, int32_t row_count,
                        int64_t poly_count);
int32_t hecuda_poly_neg(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count, int64_t poly_count);
int32_t hecuda_poly_mul_scalars(const hecuda_context *ctx, int32_t base, uint64_t *data, const uint64_t *scalars,
                                int32_t row_count, int64_t poly_count);
int32_t hecuda_poly_add_device(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs,
                               int32_t row_count, int64_t poly_count, void *stream);
int32_t hecuda_poly_sub_device(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs,
                               int32_t row_count, int64_t poly_count, void *stream);
int32_t hecuda_poly_mul_device(const hecuda_context *ctx, int32_t base, uint64_t *lhs, const uint64_t *rhs,
                               int32_t row_count, int64_t poly_count, void *stream);
int32_t hecuda_poly_neg_device(const hecuda_context *ctx, int32_t base, uint64_t *data, int32_t row_count,
                               int64_t poly_count, void *stream);
int32_t hecuda_poly_mul_scalars_device(const hecuda_context *ctx, int32_t base, uint64_t *data, const uint64_t *scalars,
                                       int32_t row_count, int64_t poly_count, void *stream);

/* ---- wire format of RNS polynomials (SURVEY.md section 8f, rank 4) ----
 * PolyRq.serialize(skipLSBs:) / PolyRq.load(from:skipLSBs:) -- PolyRq/PolyRq+Serialize.swift:28-84 over
 * CoefficientPacking.coefficientsToBytes / bytesToCoefficients (CoefficientPacking.swift:59-217): row i is a big-endian
 * bit stream of N fields of ceil(log2 q_i) - skip_lsbs bits padded to a byte, rows concatenated;
 * hecuda_poly_serialized_byte_count = PolyContext.serializationByteCount.  in / out: poly_count x row_count x N words
 * under `base`; serialized: poly_count x byte_count bytes.  Loading sets the skipped low bits to zero, as the reference. */
int32_t hecuda_poly_serialized_byte_count(const hecuda_context *ctx, int32_t base, int32_t row_count, int32_t skip_lsbs,
                                          uint64_t *bytes);
int32_t hecuda_poly_serialize(const hecuda_context *ctx, int32_t base, const uint64_t *in, int32_t skip_lsbs,
                              uint8_t *serialized, int32_t row_count, int64_t poly_count);
int32_t hecuda_poly_load(const hecuda_context *ctx, int32_t base, const uint8_t *serialized, int32_t skip_lsbs, uint64_t *out,
                         int32_t row_count, int64_t poly_count);
int32_t hecuda_poly_serialize_device(const hecuda_context *ctx, int32_t base, const uint64_t *in, int32_t skip_lsbs,
                                     uint8_t *serialized, int32_t row_count, int64_t poly_count, void *stream);
int32_t hecuda_poly_load_device(const hecuda_context *ctx, int32_t base, const uint8_t *serialized, int32_t skip_lsbs,
                                uint64_t *out, int32_t row_count, int64_t poly_count, void *stream);

/* Seeded ciphertexts.  hecuda_poly_random_from_seed = PolyRq.random(context:using:) with NistAes128Ctr(seed:)
 * (PolyRq/PolyRq+Randomize.swift:29-81; Random/NistAes128Ctr.swift, NistCtrDrbg.swift: NIST SP 800-90A CTR_DRBG over
 * AES-128 without derivation function, 4096-byte buffered): seeds batch x 32 bytes -> out batch x moduli_count x N
 * residues, coefficient k of row r = the (r N + k)-th little-endian 128-bit word of the stream mod q_r.
 * hecuda_ciphertext_expand_seeded = Ciphertext(deserialize: .seeded(poly0:seed:)) (SerializedCiphertext.swift:41-60):
 * poly0 batch x serialized bytes (hecuda_poly_serialized_byte_count, skipLSBs 0) and the seeds -> batch x 2 x
 * moduli_count x N Coeff ciphertexts (poly1 = the random polynomial, sampled in Eval format, converted to Coeff). */
int32_t hecuda_poly_random_from_seed(const hecuda_context *ctx, const uint8_t *seeds, int32_t moduli_count, uint64_t *out,
                                     int64_t batch);
int32_t hecuda_ciphertext_expand_seeded(const hecuda_context *ctx, const uint8_t *poly0, const uint8_t *seeds,
                                        int32_t moduli_count, uint64_t *out, int64_t batch);

/* Bfv.decryptCoeff -- Bfv/Bfv+Decrypt.swift:21-41 (dotProduct(ciphertext:with:) :188-204) with RnsTool.scaleAndRound
 * (RnsTool.swift:272-302).  secret_key: SecretKey.poly, (L+1) x N in Eval format (only its first moduli_count rows are
 * read); ciphertexts: batch x poly_count x moduli_count x N (Coeff, poly_count 2 or 3, any level); scaling_factor =
 * correctionFactor^-1 mod t (1 for BFV ciphertexts produced here).  plaintexts: batch x N coefficients in [0, t).
 * Client-side operation: provided so that responses can be checked where they are produced; the key copy on the device
 * is zeroized before it is freed. */
int32_t hecuda_bfv_decrypt(const hecuda_context *ctx, const uint64_t *secret_key, const uint64_t *ciphertexts,
                           int32_t poly_count, int32_t moduli_count, uint64_t scaling_factor, uint64_t *plaintexts,
                           int64_t batch);

/* Bookkeeping for bench.py: number of kernel launches issued by this library in the calling process so far. */
uint64_t hecuda_kernel_launch_count(void);

/* ---- Bfv<UInt32> data path: uint32_t buffers, context from hecuda_context_create_u32 (else INVALID_ARGUMENT).
 * Each mirrors the uint64_t entry point of the same name (same shapes, same errors). */
int32_t hecuda_u32_ntt_forward(const hecuda_context *ctx, int32_t base, uint32_t *data, int32_t row_count, int64_t poly_count);
int32_t hecuda_u32_ntt_inverse(const hecuda_context *ctx, int32_t base, uint32_t *data, int32_t row_count, int64_t poly_count);
int32_t hecuda_u32_bfv_multiply(const hecuda_context *ctx, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out, int64_t batch);
int32_t hecuda_u32_evk_create(const hecuda_context *ctx, const uint32_t *relin_key, hecuda_evk **out);
int32_t hecuda_u32_bfv_relinearize(const hecuda_context *ctx, const hecuda_evk *evk, const uint32_t *ct3, int32_t moduli_count,
                                   uint32_t *out, int64_t batch);
int32_t hecuda_u32_bfv_mod_switch_down(const hecuda_context *ctx, const uint32_t *ct, int32_t poly_count, int32_t moduli_count,
                                       uint32_t *out, int64_t batch);
int32_t hecuda_u32_bfv_multiply_relinearize(const hecuda_context *ctx, const hecuda_evk *evk, const uint32_t *lhs,
                                            const uint32_t *rhs, int32_t mod_switch, uint32_t *out, int64_t batch);
int32_t hecuda_u32_bfv_relinearize_mod_switch_down(const hecuda_context *ctx, const hecuda_evk *evk, const uint32_t *ct3,
                                                   int32_t moduli_count, uint32_t *out, int64_t batch);
int32_t hecuda_u32_evk_set_galois_key(hecuda_evk *evk, uint32_t element, const uint32_t *key);
int32_t hecuda_u32_bfv_apply_galois(const hecuda_context *ctx, const hecuda_evk *evk, const uint32_t *ct, int32_t moduli_count,
                                    uint32_t element, uint32_t *out, int64_t batch);
int32_t hecuda_u32_bfv_inner_product(const hecuda_context *ctx, const uint32_t *lhs, const uint32_t *rhs, uint32_t *out,
                                     int64_t pair_count, int64_t group_count);
int32_t hecuda_u32_rnstool_lift_q_to_qbsk(const hecuda_context *ctx, const uint32_t *polys, uint32_t *out, int64_t poly_count);
int32_t hecuda_u32_rnstool_floor_qbsk_to_q(const hecuda_context *ctx, const uint32_t *polys, uint32_t *out, int64_t poly_count);
int32_t hecuda_u32_bfv_encode_simd(const hecuda_context *ctx, const uint32_t *values, int32_t value_count,
                                   int32_t moduli_count, uint32_t *out, int64_t count);
int32_t hecuda_u32_bfv_decode_simd(const hecuda_context *ctx, const uint32_t *plaintexts, int32_t moduli_count,
                                   uint32_t *values, int64_t count);
int32_t hecuda_u32_bfv_plaintext_translate(const hecuda_context *ctx, const uint32_t *ct, int32_t poly_count,
                                           int32_t moduli_count, const uint32_t *plaintexts, int64_t plaintext_count,
                                           int32_t op, uint32_t *out, int64_t batch);

#ifdef __cplusplus
}
#endif
#endif /* HECUDA_H */
