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
 *     synchronizing.  Every kernel and copy of a `_device` call runs on `stream`, and its scratch is allocated and
 *     freed stream-ordered there (cudaMallocAsync / cudaFreeAsync), so the calls can be captured into a CUDA graph;
 *     make one call with a shape before capturing it (the first call sets kernel attributes).  Device buffers must
 *     be 16-byte aligned (the TMA row copies and the 16-byte vector loads rely on it; cudaMalloc and torch give
 *     256-byte alignment).  Exceptions are stated at the entry point (hecuda_poly_mul_scalars_device takes its
 *     scalars on the host).
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
                                  auxiliary primes are below 2^30 or 2^55 when BEHZ's exactness conditions for one product
                                  allow, else they are Bsk (as for n_8192_logq_3x55_logt_42, whose t is too large); the
                                  product does not depend on the choice (csrc/context.cu).  hecuda_bfv_inner_product uses
                                  this base only while its pair count keeps the sum exact in it, and Bsk above that.
                                  HECUDA_AUX_BASE=reference in the environment forces Bsk. */
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
/* EvaluationKey(deserialize:context:) -- SerializedKeys.swift:141-157, every key ciphertext .seeded(poly0:seed:)
 * (SerializedCiphertext.swift:126-154; encryptZero keeps its seed, Bfv+Keys.swift:69-103).  B =
 * hecuda_poly_serialized_byte_count(ctx, HECUDA_BASE_KEYSWITCH, L+1, 0).  relin_poly0: L x B, relin_seeds: L x 32
 * (both NULL = no relinearization key); galois_poly0: element_count x L x B, galois_seeds: element_count x L x 32, in the
 * order of elements[].  The DRBG expansion of `a` over [q_0..q_{L-1}, q_ks] and the unpacking of poly0 run on the device
 * and write the key buffers directly (Eval format: no NTT).  The result is an ordinary evaluation key.  It returns once
 * the keys are written.  HECUDA_ERR_UNSUPPORTED with a single coefficient modulus; HECUDA_ERR_INVALID_ARGUMENT when exactly
 * one of relin_poly0 / relin_seeds is NULL, for a negative element_count or NULL Galois arrays, and for an invalid or
 * repeated element.  On error *out is NULL.  A Bfv<UInt32> context takes the same bytes. */
int32_t hecuda_evk_create_serialized(const hecuda_context *ctx, const uint8_t *relin_poly0, const uint8_t *relin_seeds,
                                     const uint32_t *elements, int32_t element_count, const uint8_t *galois_poly0,
                                     const uint8_t *galois_seeds, hecuda_evk **out);
/* Many clients' seeded evaluation keys in one call: hecuda_evk_create_serialized for key_count clients that share one
 * EvaluationKeyConfig (a relinearization key for all or for none, the same elements[]).  With C = (has_relin +
 * element_count) x L key ciphertexts per key, client j's poly0[j] is C x B bytes and seeds[j] C x 32 bytes, the
 * relinearization key first and then elements[] in order (hecuda_evk_create_serialized's relin and Galois arrays back
 * to back).  Each client's bytes stay in the caller's own buffer.  out[j] is an ordinary, independent evaluation key;
 * the handles may be destroyed in any order, each freeing its own device memory.  A key is one device allocation that
 * holds its relinearization key (allocated even when has_relin is 0) and its Galois keys.
 * On the device: one upload of every seed and one DRBG chain launch over all key_count x C seeds, then per group of at
 * most HECUDA_EVK_LOAD_GROUP keys an upload of the group's poly0 bytes and one expansion launch; the next group's
 * upload overlaps the current group's expansion.  A group also holds at most HECUDA_EVK_LOAD_GROUP_BYTES of poly0 bytes
 * (but at least one key), which bounds the staging of contexts with large keys.  So a call makes 1 + groups kernel
 * launches whatever element_count is, and none when C = 0.  Each poly0[j] is one copy: by DMA directly when it is
 * pinned (hecuda_host_alloc, hecuda_host_register), through the driver's pinned staging when it is pageable.  The call
 * returns once every key is written.  Errors as hecuda_evk_create_serialized, plus HECUDA_ERR_INVALID_ARGUMENT for
 * key_count < 1, null out, and (when C > 0) null poly0 / seeds or a null poly0[j] / seeds[j] ("client <j>: null
 * argument").  Every argument is checked before anything is allocated or launched; on any error every out[j] is NULL
 * and nothing is left allocated. */
#define HECUDA_EVK_LOAD_GROUP 16
#define HECUDA_EVK_LOAD_GROUP_BYTES (64ull << 20)
int32_t hecuda_evk_create_serialized_many(const hecuda_context *ctx, int32_t key_count, int32_t has_relin,
                                          const uint32_t *elements, int32_t element_count, const uint8_t *const *poly0,
                                          const uint8_t *const *seeds, hecuda_evk **out);
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
/* The database's presence flags copied to the host: out[i] = 0 for a nil plaintext the scan skips, 1 otherwise (all 1
 * when it was created without flags).  capacity >= the database's plaintext count. */
int32_t hecuda_pir_database_present(const hecuda_pir_database *db, uint8_t *out, int64_t capacity);

/* Processed databases in the reference's file format -- ProcessedDatabase.serialize() / save(to:) and
 * ProcessedDatabase(from:context:) (IndexPir/IndexPirProtocol.swift:286-378): a version byte (1), plaintextCount as a
 * little-endian UInt32, then per plaintext a tag byte, 0 for nil or 1 followed by PolyRq.serialize() of the Eval
 * plaintext over every ciphertext modulus (ceil(log2 q_i) bits per coefficient, rows in order).  A keyword-PIR shard is
 * one such stream: its tables' plaintexts concatenated in table order (KeywordPir/KeywordPirProtocol.swift:161-171,
 * 230-239).  Whole plaintexts cross PCIe in chunks of at most 64 MB through two device staging buffers, and are unpacked
 * into (or packed from) the resident rows on the device; a caller buffer that is pinned (hecuda_host_alloc,
 * hecuda_host_register) is copied directly, a pageable one through pinned staging.  Peak device memory is the databases
 * and 2 x 64 MB.  A Bfv<UInt32> context reads and writes the same bytes.
 * hecuda_pir_databases_create_serialized: `byte_count` bytes -> `database_count` databases of plaintextCount /
 * database_count plaintexts each (1 for index PIR, hashFunctionCount for keyword PIR), out[t] word for word what
 * hecuda_pir_database_create builds from the same Eval plaintexts and flags.  Bytes after the last plaintext are ignored,
 * as the reference ignores them.  Refused with HECUDA_ERR_INVALID_ARGUMENT, every out[t] NULL and nothing left allocated:
 * a version other than 1 (invalidDatabaseSerializationVersion), a tag other than 0 or 1
 * (invalidDatabaseSerializationPlaintextTag), a header, tag or plaintext past the end or a plaintextCount that cannot
 * fit the buffer (corruptedData; the reference traps), no plaintexts (emptyDatabase), a plaintextCount that
 * database_count does not divide (invalidDatabasePlaintextCount), and -- checked on the device -- a residue >= its
 * modulus q_i (corruptedData, naming the plaintext and row; the reference accepts it, but the lazy accumulators of the
 * scans assume canonical residues).  Every refusal except the last launches no kernel.
 * hecuda_pir_databases_serialized_byte_count / _serialize: the serialization of `database_count` databases of one
 * context concatenated (one header over all of their plaintexts).  Refused: null pointers, databases of different
 * contexts, more than 2^32 - 1 plaintexts, only nil plaintexts (emptyDatabase), and a capacity below the size. */
int32_t hecuda_pir_databases_create_serialized(const hecuda_context *ctx, const uint8_t *bytes, uint64_t byte_count,
                                               int32_t database_count, hecuda_pir_database **out);
int32_t hecuda_pir_databases_serialized_byte_count(const hecuda_pir_database *const *databases, int32_t database_count,
                                                   uint64_t *bytes);
int32_t hecuda_pir_databases_serialize(const hecuda_pir_database *const *databases, int32_t database_count, uint8_t *out,
                                       uint64_t capacity, uint64_t *written);

/* MulPirServer.process(database:with:using:) -- IndexPir/MulPir.swift:433-556 (processPackEntries,
 * processSplitLargeEntries, CoefficientPacking.bytesToCoefficients with floor(log2 t) bits per coefficient) on the
 * device.  entries: the concatenated entry bytes; offsets: entry_count + 1 byte offsets (entry i = [offsets[i],
 * offsets[i+1])), or NULL when every entry is exactly entry_size bytes.  entry_size = IndexPirParameter.entrySizeInBytes,
 * encode_entry_size = IndexPirParameter.encodingEntrySize (a little-endian length prefix per entry), dims =
 * IndexPirParameter.dimensions (1 or 2).  count = chunkCount * prod(dims), chunkCount = ceil(encodedEntrySize /
 * bytesPerPlaintext).  Only the entry bytes (and offsets) cross PCIe; each thread of the packing kernel reads the
 * bytes its coefficient needs straight from them.
 * hecuda_pir_process_entries: plaintexts count x N coefficients (< t) and present[count] (0 = nil: all-zero, MulPir.swift:480,
 * 536) in process order -- what hecuda/pir.py plaintextRows computes on the host.
 * hecuda_pir_database_create_from_entries: the resident database hecuda_pir_database_create(those plaintexts,
 * eval_format = 0, present) builds, word for word, converted in slabs; peak device memory is the entries, the database
 * and one 64 MB slab.  A Bfv<UInt32> context works as with hecuda_pir_database_create.
 * Checked on the host before anything is allocated (HECUDA_ERR_INVALID_ARGUMENT, *out NULL): null pointers, dim_count,
 * decreasing offsets, an entry longer than entry_size (invalidDatabaseEntrySize), more entries (split) or packed plaintexts
 * than prod(dims) holds (invalidDatabaseEntryCount), and a wrong `count`. */
int32_t hecuda_pir_process_entries(const hecuda_context *ctx, const uint8_t *entries, const uint64_t *offsets,
                                   int64_t entry_count, int64_t entry_size, int32_t encode_entry_size,
                                   const int32_t *dims, int32_t dim_count, uint64_t *plaintexts, uint8_t *present,
                                   int64_t count);
int32_t hecuda_pir_database_create_from_entries(const hecuda_context *ctx, const uint8_t *entries, const uint64_t *offsets,
                                                int64_t entry_count, int64_t entry_size, int32_t encode_entry_size,
                                                const int32_t *dims, int32_t dim_count, hecuda_pir_database **out);

/* ---- Keyword PIR: KeywordPir/HashBucket.swift, CuckooTable.swift, KeywordPirProtocol.swift ------------------------
 * Keywords and values are passed as concatenated bytes with count + 1 byte offsets (row i = [offsets[i], offsets[i+1])).
 * Errors are HECUDA_ERR_INVALID_ARGUMENT with the reference's error name in hecuda_last_error(); on error *out is NULL
 * and nothing stays allocated. */

/* HashKeyword.hash (HashBucket.swift:264-269): hashes[i] = the first 8 bytes of SHA-256(keyword i) as a little-endian
 * UInt64, one device thread per keyword.  Keyword.shardIndex (KeywordDatabase.swift:56-62) is hashes[i] % shardCount. */
int32_t hecuda_keyword_hash(const uint8_t *keywords, const uint64_t *offsets, int64_t count, uint64_t *hashes);
/* HashKeyword.hashIndices (HashBucket.swift:221-257) of each keyword hash: out = count x hash_function_count candidate
 * bucket indices in [0, bucket_count), each retried with counters 1..10 while it repeats an earlier candidate. */
int32_t hecuda_keyword_hash_indices(const uint64_t *hashes, int64_t count, int64_t bucket_count,
                                    int32_t hash_function_count, int64_t *out);

typedef struct hecuda_cuckoo_table hecuda_cuckoo_table; /* CuckooTable, CuckooTable.swift:256-505 */
/* CuckooTableConfig (CuckooTable.swift:19-157).  fixed_bucket_count = 0 selects .allowExpansion(expansion_factor,
 * target_load_factor), otherwise .fixedSize(fixed_bucket_count).  defaultKeywordPir is {2, 100, size, 255, 1, 0, 1.1, 0.9}. */
typedef struct hecuda_cuckoo_config {
    int32_t hash_function_count;
    int64_t max_eviction_count;
    int64_t max_serialized_bucket_size;
    int32_t slot_count;       /* <= 255 (HashBucket.maxSlotCount) */
    int32_t multiple_tables;  /* one table per hash function */
    int64_t fixed_bucket_count;
    double expansion_factor;
    double target_load_factor;
} hecuda_cuckoo_config;
/* The generator behind CuckooTable's randomElement(using:) evictions, drawn through Swift's next(upperBound:).
 * COUNTER(seed) is _TestUtilities' TestRng(counter: seed) (TestUtilities.swift:45-61), which reproduces the reference's
 * tests; SPLITMIX64(seed) is the production choice (the reference's SystemRandomNumberGenerator is not reproducible). */
enum { HECUDA_CUCKOO_RNG_COUNTER = 0, HECUDA_CUCKOO_RNG_SPLITMIX64 = 1 };
typedef struct hecuda_cuckoo_summary {
    int64_t entry_count, bucket_count, buckets_per_table, empty_bucket_count;
    int64_t serialized_bytes;          /* sum of the serialized bucket sizes */
    int64_t max_serialized_bucket_size; /* the largest one: CuckooTable.maxSerializedBucketSize() */
} hecuda_cuckoo_summary;

/* CuckooTable.init(config:database:using:) (CuckooTable.swift:328-357, insert / insertLoop :386-458, expand :466-490):
 * the rows inserted in the order given.  The keywords are hashed on the device once and the candidate indices of every
 * row are computed on the device once per bucket count the placement reaches; the eviction loop itself runs on the host,
 * because the table depends on the order of the generator's draws.  The values are uploaded once and stay on the device
 * with the table.
 * One deliberate divergence: when no candidate bucket has a swap index, the reference expands the table and returns
 * without inserting the pair in hand (:455-457), losing that row; here the pair is inserted again after the expansion,
 * as the branch at :402-406 does.  The tables are identical whenever that branch is not taken.
 * Refused: invalidCuckooConfig (validate, :138-156, plus a target load factor <= 0 and, with expansion, a
 * max_eviction_count < 1, both of which the reference cannot build a table with), an unknown rng, decreasing offsets,
 * invalidHashBucketEntryValueSize (a value over 65535 bytes) and failedToConstructCuckooTable (a value too large for
 * any bucket, or a fixed-size table that overflows).  Rows repeating a keyword after the first are skipped, as in the
 * reference. */
int32_t hecuda_cuckoo_table_create(const hecuda_context *ctx, const uint8_t *keywords, const uint64_t *keyword_offsets,
                                   const uint8_t *values, const uint64_t *value_offsets, int64_t count,
                                   const hecuda_cuckoo_config *config, int32_t rng, uint64_t seed,
                                   hecuda_cuckoo_table **out);
/* The inputs of CuckooTable.summarize() (:361-373; loadFactor = Float(serialized_bytes) / Float(bucket_count *
 * maxSerializedBucketSize)) and of maxSerializedBucketSize() (:381-383). */
int32_t hecuda_cuckoo_table_summarize(const hecuda_cuckoo_table *table, hecuda_cuckoo_summary *out);
/* CuckooTable.serializeBuckets() (:376-378): bucket b's HashBucket bytes (HashBucket.swift:89-103, 176-187: slot count,
 * then per slot the keyword hash, the value length and the value) are bytes[offsets[b], offsets[b+1]).  offsets holds
 * bucket_count + 1 entries; capacity >= serialized_bytes.  The bytes are written by a device kernel. */
int32_t hecuda_cuckoo_table_serialize_buckets(const hecuda_cuckoo_table *table, uint8_t *bytes, uint64_t capacity,
                                              uint64_t *offsets);
int32_t hecuda_cuckoo_table_destroy(hecuda_cuckoo_table *table);

/* KeywordPirServer.process (KeywordPirProtocol.swift:191-247) after its IndexPirParameter: out[t] (t < hash function
 * count) is table t's MulPir database, word for word what hecuda_pir_database_create_from_entries builds from that
 * table's serialized buckets with entry_size, encode_entry_size = 0 and dims (uint32 rows on contexts whose moduli are
 * below 2^31 included).  The buckets are serialized on the device and each table's slice of them is packed and converted
 * to Eval there: bucket bytes never cross PCIe.  Needs a table built with multiple_tables (KeywordPirConfig,
 * :75-77: invalidCuckooConfig otherwise) and the context the table was built on.  Answer with
 * hecuda_mulpir_compute_response* over the hash-function-count databases with indices_count = hash function count. */
int32_t hecuda_keyword_pir_databases_create(const hecuda_context *ctx, const hecuda_cuckoo_table *table,
                                            int64_t entry_size, const int32_t *dims, int32_t dim_count,
                                            hecuda_pir_database **out);

/* ---- Symmetric keyword PIR: SymmetricPir/SymmetricPirDatabase.swift, config OPRF_P384_AES_GCM_192_NONCE_96_TAG_128 ----
 * The OPRF is RFC 9497 in VOPRF mode over P384-SHA384 (swift-crypto's P384._VOPRF): HashToGroup is RFC 9380
 * P384_XMD:SHA-384_SSWU_RO_ with DST "HashToGroup-" || contextString, contextString = "OPRFV1-" || 0x01 || "-P384-SHA384"
 * as RFC 9497 writes it.  The secret key is 48 big-endian bytes k with 0 < k < n (OprfPrivateKey(rawRepresentation:)).
 * These calls need no context.  Refused with HECUDA_ERR_INVALID_ARGUMENT and no kernel launched: null pointers, a
 * negative count, decreasing offsets, a key outside [1, n - 1], and an OPRF input (keyword) over 65535 bytes (its length
 * is hashed as I2OSP(len, 2)).  A count of 0 launches nothing.  The device copies of the key's recoding and of each
 * row's OPRF output are zeroized before they are freed. */
#define HECUDA_OPRF_KEY_BYTES 48
#define HECUDA_OPRF_ELEMENT_BYTES 49
#define HECUDA_OPRF_OUTPUT_BYTES 48
/* SymmetricPirConfig.clientConfig().serverPublicKey (SymmetricPirDatabase.swift:176-183): k G, SEC1 compressed. */
int32_t hecuda_oprf_public_key(const uint8_t *secret_key, uint8_t *public_key /* 49 */);
/* OprfPrivateKey.evaluate (RFC 9497 3.3.1 Evaluate) of every input, one device thread each: outputs[i] =
 * SHA-384(I2OSP(len, 2) || input || I2OSP(49, 2) || k HashToGroup(input) || "Finalize"). */
int32_t hecuda_oprf_evaluate(const uint8_t *secret_key, const uint8_t *inputs, const uint64_t *offsets, int64_t count,
                             uint8_t *outputs /* 48 * count */);
/* KeywordDatabase.symmetricPIRProcess(database:config:) (SymmetricPirDatabase.swift:193-211): with h the OPRF output of
 * keyword i, keywords_out[i] = h[0:16] and value i becomes AES.GCM.seal(value, key h[24:48], nonce h[0:12]) as ciphertext
 * || 16-byte tag, at values_out + value_offsets[i] + 16 i (value_offsets[count] + 16 count bytes in all). */
int32_t hecuda_symmetric_pir_process(const uint8_t *secret_key, const uint8_t *keywords, const uint64_t *keyword_offsets,
                                     const uint8_t *values, const uint64_t *value_offsets, int64_t count,
                                     uint8_t *keywords_out /* 16 * count */, uint8_t *values_out);
/* OprfServer.computeResponse(query:) (SymmetricPir/SymmetricPirProtocol.swift:39-59), swift-crypto's
 * P384._VOPRF.PrivateKey.evaluate: RFC 9497 3.3.2 BlindEvaluate with the 2.2.1 DLEQ proof (ComputeCompositesFast) over
 * one element, for each of `count` blinded elements, one device thread each.  responses[i] = SerializeElement(k B_i) ||
 * I2OSP(c, 48) || I2OSP(s, 48), the layout BlindEvaluation(rawRepresentation:) takes (ApplicationProtobuf/
 * PirConversion.swift:358-377).  The proof nonce is r = OS2IP(expand_message_xmd(I2OSP(k, 48) || seed || Ser(B_i),
 * "HECUDA-ProofNonce-" || contextString, 72)) mod n instead of the RFC's random draw: a verifier accepts any r in
 * [1, n - 1], and equal (k, B) give equal proofs whatever the seed, so a repeated seed cannot reuse r under two
 * challenges.  A query that is not a valid SEC1-compressed point (prefix 2 or 3, x < p, on the curve) gets status[i] = 1
 * and 145 zero bytes; the others are answered.  Refused with no kernel launched: null pointers, count < 0 and a key
 * outside [1, n - 1]. */
#define HECUDA_OPRF_PROOF_BYTES 96
#define HECUDA_OPRF_RESPONSE_BYTES 145 /* evaluated element || c || s */
#define HECUDA_OPRF_SEED_BYTES 32
int32_t hecuda_oprf_blind_evaluate(const uint8_t *secret_key, const uint8_t *blinded_elements /* count x 49 */,
                                   int64_t count, const uint8_t *seed /* 32 */,
                                   uint8_t *responses /* count x 145 */, uint8_t *status /* count: 0 ok, 1 invalid */);

/* ---- The OPRF client: OprfClient (SymmetricPir/SymmetricPirProtocol.swift:62-133), one device thread per query ----
 * swift-crypto's P384._VOPRF.PublicKey.blind and .finalize (RFC 9497 3.3.2 Blind and Finalize, with 2.2.2 VerifyProof
 * over one element), and the AES-GCM-192 open of a retrieved entry.  Blinds are 48 big-endian bytes r with 0 < r < n,
 * drawn by the caller.  These calls need no context.  Refused with HECUDA_ERR_INVALID_ARGUMENT and no kernel launched:
 * null pointers, a negative count, decreasing offsets and an OPRF input over 65535 bytes.  A count of 0 launches nothing
 * once the arguments pass.  The device copies of the blinds, the OPRF outputs and the opened values are zeroized before
 * they are freed. */
/* queryContext(at:) (:98-104): queries[i] = SerializeElement(r_i HashToGroup(input_i)) and status[i] = 0, or 49 zero
 * bytes and status[i] = 1 when r_i is not in [1, n - 1]. */
int32_t hecuda_oprf_blind(const uint8_t *inputs, const uint64_t *offsets, int64_t count,
                          const uint8_t *blinds /* count x 48 */, uint8_t *queries /* count x 49 */,
                          uint8_t *status /* count */);
/* parse(oprfResponse:with:) (:106-117), RFC 9497 VOPRF Finalize of each query: verify the response's proof against the
 * server's public key and the query, unblind the evaluated element D as N = r^-1 D, and outputs[i] = SHA-384(I2OSP(len,
 * 2) || input || I2OSP(49, 2) || Ser(N) || "Finalize").  status[i]: 0 verified and written; 1 response rejected (D not
 * a valid encoding, c >= n or s >= n, or the challenge does not match); 2 context invalid (the blind not in [1, n - 1]
 * or the query not a valid encoding).  A non-zero status writes 48 zero bytes.  A public key that is not a valid
 * SEC1-compressed point is refused with HECUDA_ERR_INVALID_ARGUMENT. */
int32_t hecuda_oprf_finalize(const uint8_t *public_key /* 49 */, const uint8_t *inputs, const uint64_t *offsets,
                             int64_t count, const uint8_t *blinds /* count x 48 */, const uint8_t *queries /* count x 49 */,
                             const uint8_t *responses /* count x 145 */, uint8_t *outputs /* count x 48 */,
                             uint8_t *status /* count */);
/* decrypt(encryptedEntry:with:) (:119-132): entry i is sealed[sealed_offsets[i] : sealed_offsets[i + 1]], ciphertext ||
 * 16-byte tag, opened with AES.GCM.open under key h[24:48] and nonce h[0:12] of oprf_outputs[i].  values has the layout
 * of sealed (sealed_offsets[count] bytes): entry i's plaintext at values[sealed_offsets[i] : sealed_offsets[i + 1] - 16]
 * and zeros in its last 16 bytes, status[i] = 0.  When the tag does not match, or the entry is shorter than 16 bytes,
 * status[i] = 1 and all of entry i's bytes in values are zero; no unauthenticated plaintext is written. */
int32_t hecuda_symmetric_pir_open(const uint8_t *oprf_outputs /* count x 48 */, const uint8_t *sealed,
                                  const uint64_t *sealed_offsets, int64_t count, uint8_t *values, uint8_t *status);

/* ---- SimplePIR: Sources/PrivateInformationRetrieval/SimplePir/ ----
 * SimplePirServer<Scalar> with Scalar = UInt32 (word_bits 32) or UInt64 (word_bits 64): requests, responses, the hint and
 * the processed database cross the boundary as little-endian words of that width.  These calls need no context; the
 * hint's single-modulus context over nttFriendlyMod (the smallest NTT prime of ct + 1 bits for degree N,
 * SimplePirContext.swift:78-81) is built inside hecuda_simple_pir_process.  The processed database DB' is columnSize (M)
 * x databaseColumns (K) and stays on the device as ceil(pt / 8) planes of u8 digits.  Every parameter the reference
 * derives is rechecked before anything is allocated (SimplePir.swift:47-79, :144-155): N a power of two, ct > pt,
 * entriesPerColumn == 1 || chunksPerEntry == 1, positive sizes -> HECUDA_ERR_INVALID_ARGUMENT; ct + 1 above word_bits
 * (generatePrimes fails there), nttFriendlyMod >= 2^62 (ct > 61) or N > 2^15 -> HECUDA_ERR_UNSUPPORTED.  Null pointers
 * and negative counts are refused with no kernel launched.  The security bound maxLog2CoefficientModulus
 * (EncryptionParameters.swift:192-219) is checked by the Python layer (hecuda.simple_pir.SimplePirEncryptionParams). */
typedef struct hecuda_simple_pir_database hecuda_simple_pir_database; /* SimplePirServer's processedDatabase, resident */
typedef struct hecuda_simple_pir_params {                            /* SimplePirParameters (SimplePir.swift:95-160) */
    int32_t plaintext_modulus_bits;  /* pt */
    int32_t ciphertext_modulus_bits; /* ct */
    int64_t lattice_dimension;       /* N */
    int64_t entry_size;              /* entrySizeInBytes */
    int64_t entries_per_column;
    int64_t chunks_per_entry;
    int64_t database_columns;        /* K */
    int32_t word_bits;               /* 32 or 64: the Scalar type */
    double error_std_dev;            /* errorStdDev: read by the client calls only (3.2 or 6.4 in the reference) */
} hecuda_simple_pir_params;
/* SimplePirServer.process(database:encryptionParams:seed:) (SimplePir+Database.swift:252-290) after computingParams
 * (:208-243): entries entry_count x entry_size bytes; seed 32 bytes (params.seed).  Entry e's bytesToCoefficients at pt
 * bits go to e * paddedEntrySize of the K x M matrix, which is transposed to DB' (M x K) and kept on the device as *out.
 * hint (M x N words) = DB' . A mod nttFriendlyMod, A the stacked negacyclic matrices of the aPolyCount = ceil(K / N)
 * polynomials PolyRq.random draws from NistAes128Ctr(seed) (:177-206); computed through the NTT without materialising A.
 * Refused: entry_count < 1, or entries that do not fit K x M (HECUDA_ERR_INVALID_ARGUMENT). */
int32_t hecuda_simple_pir_process(const uint8_t *entries, int64_t entry_count, const hecuda_simple_pir_params *params,
                                  const uint8_t *seed, void *hint, hecuda_simple_pir_database **out);
/* SimplePirServer(processedDatabase:hint:params:) (SimplePir+Server.swift:24-29): processed is DB', M x K words.  A value
 * >= 2^pt is refused with HECUDA_ERR_INVALID_ARGUMENT (the digit planes hold pt bits; process never produces one). */
int32_t hecuda_simple_pir_database_create(const void *processed, const hecuda_simple_pir_params *params,
                                          hecuda_simple_pir_database **out);
/* SimplePirDatabase.database (for save(to:), SimplePir+Database.swift:95-121): DB' as M x K words. */
int32_t hecuda_simple_pir_database_export(const hecuda_simple_pir_database *database, void *processed);
int32_t hecuda_simple_pir_database_destroy(hecuda_simple_pir_database *database);
/* SimplePirServer.computeResponse(to:) (SimplePir+Server.swift:31-38, Array2d.multiply(transposing:mask:),
 * SimplePir+Precompute.swift:51-114) for `count` requests at once: requests count x chunksPerEntry x K words, responses
 * count x chunksPerEntry x M words, response i = transpose((DB' . request_i^T) mod 2^ct).  Request bits at or above ct do
 * not change the result, as in the reference.  The _device variant follows the conventions above (stream order,
 * stream-ordered scratch, graph capture, 16-byte alignment). */
int32_t hecuda_simple_pir_compute_response(const hecuda_simple_pir_database *database, const void *requests, int64_t count,
                                           void *responses);
int32_t hecuda_simple_pir_compute_response_device(const hecuda_simple_pir_database *database, const void *requests,
                                                  int64_t count, void *responses, void *stream);
/* Sharded SimplePIR, as the SimplePIRProcessDatabase tool deploys it (Sources/SimplePIRProcessDatabase/main.swift:
 * 158-253).  DatabaseMap.shardDatabase (SimplePir/DatabaseMap.swift:82-110) cuts entry i, bytes [offsets[i],
 * offsets[i + 1]) of values, into ceil(size / chunk_size) chunks, each zero-padded to chunk_size, and puts chunk c on
 * row chunk_locations[2 j + 1] of shard chunk_locations[2 j], with j counting chunks entry-major (DatabaseMap's
 * ChunkLocation(shardIndex, index)).  The caller chooses the locations; the library draws no permutation.  Each shard
 * is then processed as hecuda_simple_pir_process would process its rows: params[s] (shard_count of them, from
 * computingParams over the shard's row count and chunk_size) and seeds[32 s .. 32 s + 32).  out[s] gets shard s's
 * resident database; hints gets every shard's hint, shard after shard, each M_s x N words.  The values cross PCIe once
 * and the shards' rows are gathered on the device.  Refused with HECUDA_ERR_INVALID_ARGUMENT before anything is
 * allocated or launched: null pointers, entry_count < 0, shard_count < 1, chunk_size < 1, decreasing offsets,
 * locations that are not a permutation of every shard's rows, a shard with no rows, params[s].entry_size !=
 * chunk_size, databaseColumns that do not match the shard's row count, and shards whose pt, ct, N or word_bits
 * differ; and every refusal of hecuda_simple_pir_process's parameters. */
int32_t hecuda_simple_pir_process_shards(const uint8_t *values, const uint64_t *offsets /* entry_count + 1 */,
                                         int64_t entry_count, int64_t chunk_size, int32_t shard_count,
                                         const int64_t *chunk_locations /* chunks x 2 */,
                                         const hecuda_simple_pir_params *params, const uint8_t *seeds /* 32 x shards */,
                                         void *hints, hecuda_simple_pir_database **out /* shard_count */);
/* computeResponse on every shard for `count` clients (SimplePirClientForAllShards.query, SimplePir+Shards.swift:
 * 47-173, sends requests_per_shard = ShardMap.chunksPerShard requests to every shard).  requests are client-major: a
 * client's block is shard 0's requests_per_shard x chunksPerEntry_0 x K_0 words, then shard 1's, and so on; responses
 * follow the same order with M_s in place of K_s.  Each response equals hecuda_simple_pir_compute_response's.  One call
 * makes one scratch allocation, one memset, one digit-split and one response launch per group of at most 32 shards,
 * and one finish launch, whatever the shard count.  Refused with no kernel launched: null pointers, shard_count < 1,
 * requests_per_shard < 1, count < 0, and shards that differ in ct or word_bits or live on different devices.
 * count == 0 launches nothing.  The _device variant follows the conventions above. */
int32_t hecuda_simple_pir_compute_response_shards(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                  int64_t requests_per_shard, const void *requests, int64_t count,
                                                  void *responses);
int32_t hecuda_simple_pir_compute_response_shards_device(const hecuda_simple_pir_database *const *shards,
                                                         int32_t shard_count, int64_t requests_per_shard,
                                                         const void *requests, int64_t count, void *responses,
                                                         void *stream);

/* ---- SimplePIR in the reference's protobuf messages (simple_pir_proto.hpp) ----
 * Requests as the reference's clients send them and responses as they expect them: api.pir.v1.SimplePIRRequest
 * { 1 request (pir.v1.SimplePIRMatrix { 1 row_count  2 col_count  3 data, repeated uint64 row-major })  2 shard_index
 * 3 configuration_hash } and api.pir.v1.SimplePIRResponse { 1 response (SimplePIRMatrix) } (api/pir/v1/pir.proto,
 * Array2d.proto() / SimplePIRMatrix.native(), PirConversion.swift:380-401).  The walks refuse what the PIR walks refuse
 * (groups, varints over 10 bytes, lengths past their message, a singular message given twice, a known field of the wrong
 * wire type); uint32 fields keep the low 32 bits of their varint.  `data` may be packed, packed in several runs, or
 * unpacked; every form answers alike.
 *
 * hecuda_simple_pir_request_fields_read: the walk of a SimplePIRRequest (host only; data is located, not read): whether
 * request is set, its row and column counts, shard_index, the number of data runs (a packed run, or one unpacked
 * element) and their bytes, and the byte range of configuration_hash (the library does not check it; nor does the
 * reference). */
typedef struct hecuda_simple_pir_request_fields {
    int32_t has_request;
    uint32_t row_count, col_count, shard_index;
    int64_t data_run_count;
    uint64_t data_bytes;
    uint64_t configuration_hash_offset, configuration_hash_bytes;
} hecuda_simple_pir_request_fields;
int32_t hecuda_simple_pir_request_fields_read(const uint8_t *bytes, uint64_t byte_count,
                                              hecuda_simple_pir_request_fields *fields);
/* The walk of `count` SimplePIRRequests against shards (as hecuda_simple_pir_compute_response_proto refuses them) and
 * each response's capacity: the SimplePIRResponse of row_count x M_s values below 2^ct, each varint ceil(ct / 7) bytes
 * long, framed as SwiftProtobuf frames it.  Values are uniform below 2^ct, so actual lengths come close to it. */
int32_t hecuda_simple_pir_response_proto_byte_count(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                    const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                    int64_t count, uint64_t *capacities);
/* SimplePirServer.computeResponse(to:) (SimplePir+Server.swift:31-38) for `count` SimplePIRRequests, each to the shard
 * its shard_index names, answered with SimplePIRResponses: message j's response is written at out + out_offsets[j]
 * (slots of at least hecuda_simple_pir_response_proto_byte_count's capacity, in order) and is out_lengths[j] bytes
 * long.  Its data equals hecuda_simple_pir_compute_response's for the message's row_count x K_s words, row-major; a
 * message with row_count 0 gets an empty 0 x M_s matrix (col_count M_s, no data).  The shards must share ct and
 * ceil(pt / 8); their word sizes may differ.
 *
 * Refused on the host, with nothing enqueued, each refusal naming its message ("message <j>: "): every walk refusal
 * above, an unset request, shard_index >= shard_count, col_count != the shard's databaseColumns (the reference's
 * precondition traps there), and more rows to one shard than 2^36 / max(K_s, M_s).  Refused on the device, naming the
 * first bad message and leaving out and out_lengths untouched: a data varint longer than 10 bytes, one that runs past its
 * run, a value >= 2^32 to a 32-bit shard (the reference's Scalar(_:) traps there), and a varint count other than
 * row_count x col_count.  Request bits at or above ct are ignored, as in the reference.
 *
 * The messages cross PCIe as they are.  On the device, a scan over the varints' last bytes places every value, which is
 * decoded straight into its shard's request digit planes; all rows to one shard form its query block for one grouped
 * response launch per group of at most 32 shards that have rows; the responses are encoded straight from the
 * accumulators (lengths, a scan of them, then every message whole).  A call makes four decode launches, the response
 * launches and three encode launches, however many messages it has. */
int32_t hecuda_simple_pir_compute_response_proto(const hecuda_simple_pir_database *const *shards, int32_t shard_count,
                                                 const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                 int64_t count, uint8_t *out, const uint64_t *out_offsets,
                                                 uint64_t *out_lengths);
/* Client side, host only.  hecuda_simple_pir_request_write: Array2d.proto() of row_count x col_count words (data, as
 * uint64) in a SimplePIRRequest with shard_index and configuration_hash (omitted when hash_bytes is 0), data packed.
 * With out NULL only *written is set; else capacity must hold it.  hecuda_simple_pir_response_read: a SimplePIRResponse's
 * dimensions and its row_count x col_count values (at most capacity; refused when the count differs). */
int32_t hecuda_simple_pir_request_write(uint32_t row_count, uint32_t col_count, const uint64_t *data, uint32_t shard_index,
                                        const uint8_t *configuration_hash, uint64_t hash_bytes, uint8_t *out,
                                        uint64_t capacity, uint64_t *written);
int32_t hecuda_simple_pir_response_read(const uint8_t *bytes, uint64_t byte_count, uint32_t *row_count, uint32_t *col_count,
                                        uint64_t *data, int64_t capacity);
/* api.pir.v1.SimplePIRConfig as the SimplePIRProcessDatabase tool writes it (main.swift:193-258): pir.v1.DatabaseMapping
 * { 1 entries { 1 original_index  2 size  3 chunks { 1 shard_index  2 index } }  2 chunk_size }, one
 * pir.v1.SimplePIRParameters per shard { 1 encryption_params { 1 lattice_dimension  2 error_std_dev (double)
 * 3 plaintext_bits  4 ciphertext_bits }  2 a_seed  3 entry_size_in_bytes  4 entries_per_column  5 chunks_per_entry
 * 6 database_columns }, and one hint identifier per shard (SHA-256 of the hint file) -- DatabaseMap.proto() and
 * SimplePirParameters.proto() / native() (PirConversion.swift:403-518).
 * hecuda_simple_pir_config_describe: the counts, after every refusal: the walk's, an errorStdDev other than 3.2 or 6.4
 * and an a_seed that is not 32 bytes (as native() refuses), and every refusal of hecuda_simple_pir_process's
 * parameters, with word_bits 32 for ct <= 32 and 64 otherwise (main.swift:369-371).  hecuda_simple_pir_config_read
 * then fills: per entry its original index, size and chunk count; the chunk locations (shard, index) entry-major; each
 * shard's params and 32-byte seed; each hint identifier's (offset, length) in `bytes`.
 * hecuda_simple_pir_config_serialized_byte_count / _serialize: the same fields written as SwiftProtobuf writes them. */
typedef struct hecuda_simple_pir_config_shape {
    int64_t entry_count, chunk_count;
    uint64_t chunk_size;
    int32_t shard_count, hint_identifier_count;
} hecuda_simple_pir_config_shape;
int32_t hecuda_simple_pir_config_describe(const uint8_t *bytes, uint64_t byte_count, hecuda_simple_pir_config_shape *shape);
int32_t hecuda_simple_pir_config_read(const uint8_t *bytes, uint64_t byte_count, uint64_t *original_indices, uint64_t *sizes,
                                      uint64_t *chunk_counts, int64_t *chunk_locations, hecuda_simple_pir_params *params,
                                      uint8_t *seeds, uint64_t *hint_identifier_ranges);
int32_t hecuda_simple_pir_config_serialized_byte_count(const uint64_t *original_indices, const uint64_t *sizes,
                                                       const uint64_t *chunk_counts, int64_t entry_count,
                                                       const int64_t *chunk_locations, uint64_t chunk_size,
                                                       const hecuda_simple_pir_params *params, const uint8_t *seeds,
                                                       int32_t shard_count, const uint8_t *const *hint_identifiers,
                                                       const uint64_t *hint_identifier_bytes, int32_t hint_count,
                                                       uint64_t *bytes);
int32_t hecuda_simple_pir_config_serialize(const uint64_t *original_indices, const uint64_t *sizes,
                                           const uint64_t *chunk_counts, int64_t entry_count, const int64_t *chunk_locations,
                                           uint64_t chunk_size, const hecuda_simple_pir_params *params, const uint8_t *seeds,
                                           int32_t shard_count, const uint8_t *const *hint_identifiers,
                                           const uint64_t *hint_identifier_bytes, int32_t hint_count, uint8_t *out,
                                           uint64_t capacity);

/* SimplePIR's client (SimplePirClient with DefaultQueryGenerator, SimplePir+Client.swift, SimplePir+Precompute.swift).
 * hecuda_simple_pir_client_create: DefaultQueryGenerator.init (SimplePir+Precompute.swift:328-334) from the hint (M x N
 * words), params and seed (32 bytes, params.seed): the aPolyCount polynomials PolyRq.random draws from
 * NistAes128Ctr(seed) (generateAPolynomials, SimplePir+Database.swift:177-184) stay on the device in Eval format, and the
 * hint as ceil((ct + 1) / 8) u8 digit planes.  Refused with HECUDA_ERR_INVALID_ARGUMENT: every refusal of
 * hecuda_simple_pir_process's parameters, null pointers, a hint word >= nttFriendlyMod, errorStdDev not in (0, 16).
 * The AES tables are uploaded here, so the _device calls below stay stream-ordered and graph-capturable. */
typedef struct hecuda_simple_pir_client hecuda_simple_pir_client;
int32_t hecuda_simple_pir_client_create(const void *hint /* M x N words */, const hecuda_simple_pir_params *params,
                                        const uint8_t *seed /* 32, params.seed */, hecuda_simple_pir_client **out);
int32_t hecuda_simple_pir_client_destroy(hecuda_simple_pir_client *client);
/* PrecomputedQueries.WithoutIndices.init (SimplePir+Precompute.swift:199-227; generateSecretPolys, noiselessSample and
 * encryptZero, SimplePir+Client.swift:20-82) for `count` queries, each drawn from two 32-byte seeds (count x 32 each)
 * in place of the reference's SystemRandomNumberGenerator and rng: secret i < chunksPerEntry, coefficient j is stream
 * coefficient i N + j of PolyRq.randomizeTernary over NistAes128Ctr(secret seed) (12 bytes each, -1 stored as p - 1);
 * error (i, c) is stream coefficient i K + c of Array2d.randomCenteredBinomialDistribution over NistAes128Ctr(error seed)
 * (Array2d.swift:382-429).  queries: count x chunksPerEntry x K words, the modSwitched sample divideAndRound(p -> 2^ct)
 * plus the error, masked to ct bits; with indices (count, nullable) each query is WithQueryIndices.queries, delta =
 * 2^(ct - pt) added at column (index chunksPerEntry + i) / entriesPerColumn (add(index:), :241-256).  results: count x
 * chunksPerEntry x M words = S . hint^T mod p as Array2d.multiply(transposing:modulus:) (:122-188) computes it: the sum
 * in the scalar's double width with wrapping adds, then mod p, so results where that sum wraps are the reference's, not
 * the exact product.  Refused with no kernel launched: null pointers, count < 0, an index < 0 or whose column reaches K
 * (host variant), more than 2^40 / (chunksPerEntry max(K, M)) queries.  count == 0 launches nothing.  The _device
 * variant takes device buffers (indices too, unchecked) and follows the conventions above. */
int32_t hecuda_simple_pir_client_precompute(const hecuda_simple_pir_client *client, const uint8_t *secret_seeds,
                                            const uint8_t *error_seeds, const int64_t *indices, int64_t count,
                                            void *queries, void *results);
int32_t hecuda_simple_pir_client_precompute_device(const hecuda_simple_pir_client *client, const uint8_t *secret_seeds,
                                                   const uint8_t *error_seeds, const int64_t *indices, int64_t count,
                                                   void *queries, void *results, void *stream);
/* SimplePirClient.decrypt (SimplePir+Client.swift:111-121) after prepareResponse and integrate (SimplePir+Precompute.swift:
 * 280-311) for `count` responses (count x chunksPerEntry x M words) with the results precompute wrote for them and their
 * indices (count): extractEntries of both at the index, ((r - s + delta / 2) & mask) >> (ct - pt), coefficientsToBytes
 * at pt bits, the first entrySizeInBytes bytes -> entries (count x entrySizeInBytes).  Refusals as precompute's, indices
 * required. */
int32_t hecuda_simple_pir_client_decrypt(const hecuda_simple_pir_client *client, const void *responses, const void *results,
                                         const int64_t *indices, int64_t count, uint8_t *entries);
int32_t hecuda_simple_pir_client_decrypt_device(const hecuda_simple_pir_client *client, const void *responses,
                                                const void *results, const int64_t *indices, int64_t count,
                                                uint8_t *entries, void *stream);

/* PirUtil.expand(ciphertexts:outputCount:using:) -- IndexPir/PirUtil.swift:321-355 (expandCiphertext :249-304,
 * expandCiphertextForOneStep :204-236).  ciphertexts: ciphertext_count x 2 x L x N (Coeff); out: output_count x 2 x L x N,
 * output i encrypting the constant polynomial whose constant is coefficient i of the inputs (x 2^ceilLog2(count)).
 * The Galois keys come from `evk` (hecuda_evk_set_galois_key); the largest configured element <= 2^(logN-logStep+1)+1
 * is applied repeatedly, HECUDA_ERR_MISSING_KEY if none fits (HeError.missingGaloisKey, :216-220).
 * The MulPir _device variants (here and below) take device buffers and only enqueue on `stream`.  The first MulPir call
 * with a new query shape uploads that shape's expansion plan to the context once, synchronously: make one call with a
 * shape before capturing calls with it into a graph. */
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

/* Many clients' queries in one call: the same PirUtil.computeResponse (PirUtil.swift:490-568) that
 * MulPirServer.computeResponse (MulPir.swift:414) runs once per Query, for client_count queries of the same shape
 * against the same databases.  Client c is answered with evks[c]; its query ciphertexts are
 * queries + c * query_ciphertext_count * 2 * L * N and its reply (bit-identical to what hecuda_mulpir_compute_response
 * returns for that client alone) is out + c * indices_count * chunk_count * 2 * N, so out is
 * client_count x indices_count x chunk_count x 2 x 1 x N.  Clients are processed in groups of at most
 * HECUDA_MULPIR_CLIENT_GROUP; every stage is one pass over a group (from two clients up, its launch count does not
 * depend on the group's size), the first-dimension scan streams each database once per group, and temporaries scale
 * with the group, not with client_count.  A group of one client runs the kernels of hecuda_mulpir_compute_response.
 * Every client is checked like a single call (a failure's message names the client).  At every expansion level all
 * clients' Galois keys must resolve to the same element, as keys generated for the same IndexPirParameter do;
 * HECUDA_ERR_INVALID_ARGUMENT otherwise (answer such a client with the single-client call). */
#define HECUDA_MULPIR_CLIENT_GROUP 16
int32_t hecuda_mulpir_compute_response_clients(const hecuda_context *ctx, const hecuda_evk *const *evks, int32_t client_count,
                                               const hecuda_pir_database *const *databases, int32_t database_count,
                                               const int32_t *dimensions, int32_t dimension_count, int32_t chunk_count,
                                               const uint64_t *queries, int32_t query_ciphertext_count,
                                               int32_t indices_count, uint64_t *out);
int32_t hecuda_mulpir_compute_response_clients_device(const hecuda_context *ctx, const hecuda_evk *const *evks,
                                                      int32_t client_count, const hecuda_pir_database *const *databases,
                                                      int32_t database_count, const int32_t *dimensions,
                                                      int32_t dimension_count, int32_t chunk_count, const uint64_t *queries,
                                                      int32_t query_ciphertext_count, int32_t indices_count, uint64_t *out,
                                                      void *stream);

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

/* hecuda_mulpir_compute_response_clients on the wire: each client's bytes are what hecuda_mulpir_compute_response_wire
 * returns for that client alone.  query_poly0: client_count x query_ciphertext_count x byteCount(L rows, skipLSBs 0),
 * query_seeds: client_count x query_ciphertext_count x 32; out: client_count x indices_count x chunk_count x
 * (byteCount(1 row, skip0) + byteCount(1 row, skip1)).  Arguments are checked and keys resolved as by the two calls it
 * combines.  Per group of HECUDA_MULPIR_CLIENT_GROUP clients: one seeded expansion of all the group's query ciphertexts,
 * the many-clients response pipeline, and one packing pass per reply poly. */
int32_t hecuda_mulpir_compute_response_clients_wire(const hecuda_context *ctx, const hecuda_evk *const *evks,
                                                    int32_t client_count, const hecuda_pir_database *const *databases,
                                                    int32_t database_count, const int32_t *dimensions,
                                                    int32_t dimension_count, int32_t chunk_count, const uint8_t *query_poly0,
                                                    const uint8_t *query_seeds, int32_t query_ciphertext_count,
                                                    int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                                    uint8_t *out);

/* ---- PIR in the reference's protobuf messages (pir_proto.hpp) ----
 * Requests as the reference's clients send them and responses as they expect them: pir.v1.EncryptedIndices
 * (PirConversion.swift:23-53), v1.SerializedEvaluationKey (ConversionHe.swift) and api.pir.v1.PIRResponse
 * (PirConversionApi.swift:20-49).  A host walk of each message finds its payloads (refusing groups, varints over 10
 * bytes, lengths past their message, a singular message given twice and a known field of the wrong wire type); the
 * message then crosses PCIe as it is and the kernels read poly0 and the seeds in place.
 *
 * hecuda_pir_request_fields: the walk of an api.pir.v1.PIRRequest (host only, nothing copied): its scalar fields, and
 * the byte ranges (offsets into `bytes`) of the query (an EncryptedIndices), of evaluation_key.evaluation_key (a
 * SerializedEvaluationKey), of the configuration hash, the shard id and the key identifier.  The key metadata is
 * evaluation_key_metadata, or evaluation_key.metadata when that is absent.  Routing by shard and caching keys by
 * identifier stay the caller's. */
typedef struct hecuda_pir_request_fields {
    uint32_t shard_index;
    int32_t has_shard_id, has_query, has_evaluation_key, has_key_metadata;
    uint64_t shard_id_offset, shard_id_bytes;
    uint64_t configuration_hash_offset, configuration_hash_bytes;
    uint64_t query_offset, query_bytes;
    uint64_t evaluation_key_offset, evaluation_key_bytes;
    uint64_t key_timestamp, key_identifier_offset, key_identifier_bytes;
} hecuda_pir_request_fields;
int32_t hecuda_pir_request_fields_read(const uint8_t *bytes, uint64_t byte_count, hecuda_pir_request_fields *out);

/* EvaluationKey(deserialize:) of key_count clients' SerializedEvaluationKey messages (message j: message_byte_counts[j]
 * bytes), as hecuda_evk_create_serialized_many does for the same payloads: the galois_key map (uint64 element ->
 * SerializedKeySwitchKey of L ciphertexts, entries in any order) and the optional relin_key.  Every key ciphertext must
 * be .seeded (HECUDA_ERR_UNSUPPORTED for .full keys, which the reference's key generation does not write).  Every
 * client must resolve to client 0's configuration: a relinearization key for all or none, and the same set of Galois
 * elements in any map order; a repeated element is refused.  Every message is walked and checked before anything is
 * allocated; failures name the client ("client <j>: ").  On the device: one upload of all the messages, one DRBG chain
 * launch over every seed read in place, and one expansion launch.  On any error every out[j] is NULL and nothing is
 * left allocated. */
int32_t hecuda_evk_create_proto_many(const hecuda_context *ctx, int32_t key_count, const uint8_t *const *messages,
                                     const uint64_t *message_byte_counts, hecuda_evk **out);

/* The size of one client's PIRResponse for indices_count replies of chunk_count ciphertexts, each
 * SerializedCiphertext.full { polys = UInt16 2, poly 0 and poly 1 packed with skip_lsbs_poly0 / skip_lsbs_poly1 dropped
 * bits, skip_lsbs = [skip0, skip1], correction_factor = 1 }: Response.proto() as SwiftProtobuf writes it. */
int32_t hecuda_mulpir_response_proto_byte_count(const hecuda_context *ctx, int32_t chunk_count, int32_t indices_count,
                                                int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint64_t *bytes);

/* hecuda_mulpir_compute_response_clients_wire with one EncryptedIndices message per client in (message c:
 * message_byte_counts[c] bytes) and one PIRResponse per client out: out is client_count x
 * hecuda_mulpir_response_proto_byte_count bytes and client c's slice is a complete PIRResponse whose poly bytes are the
 * bytes hecuda_mulpir_compute_response_clients_wire returns for the same poly0 and seeds.  A query ciphertext may be
 * .seeded or .full (two polys over L rows with their skip bits, correction factor 1; any other correction factor is
 * HECUDA_ERR_UNSUPPORTED).  num_pir_calls must equal indices_count, and the ciphertext count must be the one the
 * parameter's expansion takes (hecuda_mulpir_compute_response's refusals).  Every client is walked and checked before
 * anything is enqueued; a failure's message starts with "client <c>: " and leaves `out` untouched.  Per group of
 * HECUDA_MULPIR_CLIENT_GROUP clients: one upload of the group's messages, one seeded expansion reading them in place,
 * the many-clients response pipeline, one framing launch and one packing launch per reply poly, written straight into
 * the clients' PIRResponse bytes. */
int32_t hecuda_mulpir_compute_response_clients_proto(const hecuda_context *ctx, const hecuda_evk *const *evks,
                                                     int32_t client_count, const hecuda_pir_database *const *databases,
                                                     int32_t database_count, const int32_t *dimensions,
                                                     int32_t dimension_count, int32_t chunk_count,
                                                     const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                     int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                                     uint8_t *out);

/* Client side, host only.  hecuda_pir_encrypted_indices_write: Query.proto() of ciphertext_count .seeded ciphertexts
 * (poly0: ciphertext_count x byteCount(L rows), seeds: ciphertext_count x 32) with num_pir_calls = indices_count; with
 * out NULL only *written is set to the size, else HECUDA_ERR_INVALID_ARGUMENT when capacity is below it.
 * hecuda_pir_evaluation_key_write: SerializedEvaluationKey.proto() of a seeded key in the arrays of
 * hecuda_evk_create_serialized (relin_poly0 / relin_seeds NULL: no relinearization key), map entries in elements[]
 * order.  hecuda_pir_response_read: the offsets in a PIRResponse of every reply ciphertext's poly 0 (poly 1 follows it),
 * poly_offsets[indices_count x chunk_count], refused unless it holds that many .full ciphertexts with the given skip bits
 * and one-modulus sizes. */
int32_t hecuda_pir_encrypted_indices_write(const hecuda_context *ctx, const uint8_t *poly0, const uint8_t *seeds,
                                           int32_t ciphertext_count, int32_t indices_count, uint8_t *out, uint64_t capacity,
                                           uint64_t *written);
int32_t hecuda_pir_evaluation_key_write(const hecuda_context *ctx, const uint8_t *relin_poly0, const uint8_t *relin_seeds,
                                        const uint32_t *elements, int32_t element_count, const uint8_t *galois_poly0,
                                        const uint8_t *galois_seeds, uint8_t *out, uint64_t capacity, uint64_t *written);
int32_t hecuda_pir_response_read(const hecuda_context *ctx, const uint8_t *bytes, uint64_t byte_count, int32_t chunk_count,
                                 int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                 uint64_t *poly_offsets);

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

/* PlaintextMatrix.init(context:dimensions:packing: .diagonal, signedValues:reduce:) -- PlaintextMatrix.swift:155-190 --
 * with diagonalPlaintexts (:417-482) on the device.  values: row_count x column_count signed values, row-major; each
 * becomes Modulus.reduce(value) (reduce = 1) or value.centeredToRemainder(t), which requires value in
 * [-floor(t/2), floor((t-1)/2)] (HECUDA_ERR_INVALID_ARGUMENT otherwise).  Diagonal d holds
 * data[c][(c + d) mod nextPow2(cols)] (0 past cols); each N-chunk of it has both SIMD half-rows rotated by
 * floor(d / baby_step) * baby_step and is SIMD-encoded.  One kernel does the conversion, gather, rotation and encodeSimd
 * scatter; the inverse NTT mod t follows.  HECUDA_ERR_UNSUPPORTED without SIMD support (simdEncodingNotSupported),
 * invalidMatrixDimensions when column_count > N/2.
 * hecuda_pnns_diagonal_plaintexts: out = nextPow2(cols) * ceil(rows / N) Coeff plaintexts x N, in the order
 * hecuda_pnns_matrix_create takes them (out is unspecified when a value is out of range).
 * hecuda_pnns_matrix_create_from_values: the handle hecuda_pnns_matrix_create(those plaintexts, eval_format = 0, ...)
 * builds -- the same resident words, flags and shape -- written in its slot order and converted to Eval in slabs;
 * baby_step / giant_step are checked as there.  On error *out is NULL and nothing stays allocated. */
int32_t hecuda_pnns_diagonal_plaintexts(const hecuda_context *ctx, const int64_t *values, int32_t reduce,
                                        int64_t row_count, int64_t column_count, int32_t baby_step, uint64_t *out);
int32_t hecuda_pnns_matrix_create_from_values(const hecuda_context *ctx, const int64_t *values, int32_t reduce,
                                              int64_t row_count, int64_t column_count, int32_t baby_step,
                                              int32_t giant_step, hecuda_pnns_matrix **out);
/* The resident plaintexts, [result][giant][baby] x L x N uint64 Eval words (bytes = result_count * giant * baby * L * N * 8),
 * as hecuda_pir_database_device_buffer gives a database's (device-to-device copies between ranks). */
int32_t hecuda_pnns_matrix_device_buffer(hecuda_pnns_matrix *matrix, void **device_ptr, uint64_t *bytes);
/* The matrix's presence flags in its resident slot order ([result][giant][baby]) copied to the host: 0 for a slot past
 * the padded dimension (an absent plaintext).  capacity >= result_count * giant * baby. */
int32_t hecuda_pnns_matrix_present(const hecuda_pnns_matrix *matrix, uint8_t *out, int64_t capacity);

/* ---- PNNS processed databases and configurations in the reference's protobuf format ----
 * apple.swift_homomorphic_encryption.pnns.v1.SerializedProcessedDatabase (proto3 binary): the plaintext matrices, one
 * per plaintext modulus, each plaintext PolyRq.serialize() of its L Eval rows; the entry identifiers and metadata; the
 * ServerConfig.  Saves are byte for byte what SwiftProtobuf writes (fields in field-number order, proto3 zero scalars
 * omitted, repeated scalars packed).  Loads accept any conforming encoding: fields in any order, unknown fields of wire
 * types 0, 1, 2 and 5, repeated scalars packed or not.  Refused: groups, varints over 10 bytes, lengths that run past
 * the buffer, a singular message field given twice, and a wrong wire type for a known field.
 *
 * hecuda_pnns_server_config holds a ServerConfig (or, with database_packing = 0, a ClientConfig).  Enumerations keep
 * their protobuf numbers: error_std_dev 0 = stdDev32 (3.2), 1 = stdDev64 (6.4); security_level 0 = unchecked
 * (SECURITY_LEVEL_UNSPECIFIED), 1 = quantum128; he_scheme 0 = unspecified, 1 = BFV, 2 = BGV; distance_metric 0 =
 * cosineSimilarity; a packing 0 = unset, 1 = denseRow, 2 = diagonal (with its BabyStepGiantStep), 3 = denseColumn.  A
 * message with more coefficient moduli, extra plaintext moduli or Galois elements than the arrays hold is
 * HECUDA_ERR_UNSUPPORTED. */
#define HECUDA_PNNS_MAX_COEFFICIENT_MODULI 32    /* the reference's own limit */
#define HECUDA_PNNS_MAX_EXTRA_PLAINTEXT_MODULI 7 /* 8 plaintext moduli: hecuda_pnns_decrypt_distances' limit */
#define HECUDA_PNNS_MAX_GALOIS_ELEMENTS 64
typedef struct hecuda_pnns_server_config {
    /* ClientConfig.encryption_parameters (v1.EncryptionParameters); coefficient_moduli include the key-switching one */
    uint64_t poly_degree;
    uint64_t plaintext_modulus;
    int32_t coefficient_moduli_count;
    int32_t error_std_dev;
    uint64_t coefficient_moduli[HECUDA_PNNS_MAX_COEFFICIENT_MODULI];
    int32_t security_level;
    int32_t he_scheme;
    /* the rest of ClientConfig */
    uint64_t scaling_factor;
    int32_t query_packing;
    uint32_t query_vector_dimension, query_baby_step, query_giant_step; /* query_packing = 2 only */
    uint32_t vector_dimension;
    int32_t galois_element_count;
    uint32_t galois_elements[HECUDA_PNNS_MAX_GALOIS_ELEMENTS];
    int32_t distance_metric;
    int32_t extra_plaintext_moduli_count;
    uint64_t extra_plaintext_moduli[HECUDA_PNNS_MAX_EXTRA_PLAINTEXT_MODULI];
    /* ServerConfig.database_packing */
    int32_t database_packing;
    uint32_t database_vector_dimension, database_baby_step, database_giant_step; /* database_packing = 2 only */
} hecuda_pnns_server_config;

/* A ServerConfig message (hecuda_pnns_server_config_*) or a ClientConfig message (hecuda_pnns_client_config_*) on its
 * own, as the reference's tools write them beside a database.  Parsing refuses what ServerConfig / ClientConfig.native()
 * refuses, by the reference's error names: unsetField (no client_config / encryption_parameters), unsetOneof (a packing
 * with no type), unrecognizedEnumValue, invalidScheme (BGV).  Serializing writes `*written` bytes to `out`; with out =
 * NULL it only sets *written to the size.  HECUDA_ERR_INVALID_ARGUMENT when capacity is below it. */
int32_t hecuda_pnns_server_config_parse(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *out);
int32_t hecuda_pnns_server_config_serialize(const hecuda_pnns_server_config *config, uint8_t *out, uint64_t capacity,
                                            uint64_t *written);
int32_t hecuda_pnns_client_config_parse(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *out);
int32_t hecuda_pnns_client_config_serialize(const hecuda_pnns_server_config *config, uint8_t *out, uint64_t capacity,
                                            uint64_t *written);

/* What a SerializedProcessedDatabase holds, from one walk of its framing (no payload is read, nothing is allocated on
 * the device): its ServerConfig, the number of plaintext matrices and their row and column counts (the same for every
 * matrix, or HECUDA_ERR_INVALID_ARGUMENT), the entry-identifier count, and the metadata count and total bytes.
 * hecuda_pnns_database_entries copies the identifiers (id_capacity >= their count) and the metadata: entry k's bytes are
 * metadata[metadata_offsets[k] .. metadata_offsets[k + 1]) (offsets_capacity >= count + 1).  Null buffers are skipped. */
int32_t hecuda_pnns_database_describe(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *config,
                                      int32_t *matrix_count, int64_t *row_count, int64_t *column_count,
                                      int64_t *entry_id_count, int64_t *metadata_count, uint64_t *metadata_bytes);
int32_t hecuda_pnns_database_entries(const uint8_t *bytes, uint64_t byte_count, uint64_t *entry_ids, int64_t id_capacity,
                                     uint8_t *metadata, uint64_t metadata_capacity, uint64_t *metadata_offsets,
                                     int64_t offsets_capacity);

/* ProcessedDatabase(from:contexts:) (ProcessedDatabase.swift:56-75) for its plaintext matrices, unpacked on the device:
 * out[k] is the matrix of plaintext modulus k over ctxs[k], word for word the handle hecuda_pnns_matrix_create(
 * eval_format = 1, ...) builds from the same plaintexts (the same resident words, flags, result count and steps).
 * count must equal 1 + the config's extra plaintext moduli (wrongContextsCount) and every context the config's
 * parameters (wrongEncryptionParameters); every matrix must be .diagonal (HECUDA_ERR_UNSUPPORTED otherwise), hold
 * nextPow2(num_columns) * ceil(num_rows / N) plaintexts (wrongPlaintextCount), each of exactly L serialized rows, with
 * steps hecuda_pnns_matrix_create accepts.  All of it is checked before anything is allocated.  Whole plaintexts cross
 * PCIe in chunks of at most 64 MB, through pinned staging unless `bytes` is pinned.  Residues >= their modulus are
 * refused (the reference accepts them), naming the matrix, plaintext and row.  On error every out[k] is NULL and nothing
 * stays allocated. */
int32_t hecuda_pnns_matrices_create_serialized(const hecuda_context *const *ctxs, int32_t count, const uint8_t *bytes,
                                               uint64_t byte_count, hecuda_pnns_matrix **out);
/* ProcessedDatabase.serialize() (ProcessedDatabase.swift:81-88) followed by proto().serializedData(): matrices[k] of
 * plaintext modulus k, the entry identifiers, the metadata (entry k at metadata[metadata_offsets[k] ..
 * metadata_offsets[k + 1]); metadata_count 0 for none), and `config`, whose parameters must match the matrices'
 * contexts and whose database packing must be the matrices' .diagonal steps.  The plaintexts are packed on the device
 * with their framing, so each chunk leaves as one contiguous range of the file.  *written = the byte count. */
int32_t hecuda_pnns_database_serialized_byte_count(const hecuda_pnns_matrix *const *matrices, int32_t count,
                                                   const uint64_t *entry_ids, int64_t entry_id_count,
                                                   const uint8_t *metadata, const uint64_t *metadata_offsets,
                                                   int64_t metadata_count, const hecuda_pnns_server_config *config,
                                                   uint64_t *bytes);
int32_t hecuda_pnns_database_serialize(const hecuda_pnns_matrix *const *matrices, int32_t count, const uint64_t *entry_ids,
                                       int64_t entry_id_count, const uint8_t *metadata, const uint64_t *metadata_offsets,
                                       int64_t metadata_count, const hecuda_pnns_server_config *config, uint8_t *out,
                                       uint64_t capacity, uint64_t *written);

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

/* Many PNNS clients in one call: Server.computeResponse (PrivateNearestNeighborSearch/Server.swift:61-88) for one
 * plaintext matrix -- mulTranspose(matrix:using:) + modSwitchDownToSingle -- for client_count queries of the same shape,
 * client c answered with evks[c].  ciphertexts: client_count x ciphertext_count x 2 x L x N (Coeff); the row descriptors
 * are those of hecuda_pnns_mul_transpose_matrix, shared by all clients.  out: client_count x out_capacity ciphertexts of
 * 2 x 1 x N; *out_count replies per client.  Client c's replies (out + c * out_capacity * 2 * N) are bit-identical to what
 * hecuda_pnns_mul_transpose_matrix(..., mod_switch_to_single = 1) returns for that client alone.  Clients are processed
 * in groups of at most HECUDA_PNNS_CLIENT_GROUP: every rotation is one key-switching pass over a group, each client with
 * its own keys, and the matrix streams from HBM once per group (from two clients up, the launch count does not depend
 * on the group's size); temporaries scale with the group.  A group of one runs the kernels of
 * hecuda_pnns_mul_transpose_matrix.  Every client's key is checked and every Galois key it needs found before anything
 * is enqueued (a failure's message starts with "client <c>: " and leaves out untouched); out_capacity too small:
 * HECUDA_ERR_INVALID_ARGUMENT with *out_count set to the replies needed per client. */
#define HECUDA_PNNS_CLIENT_GROUP 16
int32_t hecuda_pnns_compute_response_clients(const hecuda_context *ctx, const hecuda_evk *const *evks, int32_t client_count,
                                             const hecuda_pnns_matrix *matrix, const uint64_t *ciphertexts,
                                             int32_t ciphertext_count, int32_t query_row_count,
                                             const int32_t *row_ciphertext_index, const uint64_t *row_masks,
                                             const int32_t *row_rotate_count, int32_t column_step,
                                             const int32_t *pack_rotations, int32_t pack_rotation_count, uint64_t *out,
                                             int64_t out_capacity, int64_t *out_count);

/* The same on the wire (ApplicationProtobuf/PnnsConversionApi.swift:48): the query ciphertexts as
 * SerializedCiphertext.seeded (query_poly0: client_count x ciphertext_count x byteCount(L rows, skipLSBs 0),
 * query_seeds: client_count x ciphertext_count x 32; SerializedCiphertext.swift:41-49,126-154) and the replies serialized
 * forDecryption with skip_lsbs_poly0 / skip_lsbs_poly1 dropped bits (Bfv.skipLSBsForDecryption,
 * Bfv+Decrypt.swift:51-110).  out: client_count x out_capacity x (byteCount(1 row, skip0) + byteCount(1 row, skip1))
 * bytes.  Invalid skips: HECUDA_ERR_INVALID_ARGUMENT. */
int32_t hecuda_pnns_compute_response_clients_wire(const hecuda_context *ctx, const hecuda_evk *const *evks,
                                                  int32_t client_count, const hecuda_pnns_matrix *matrix,
                                                  const uint8_t *query_poly0, const uint8_t *query_seeds,
                                                  int32_t ciphertext_count, int32_t query_row_count,
                                                  const int32_t *row_ciphertext_index, const uint64_t *row_masks,
                                                  const int32_t *row_rotate_count, int32_t column_step,
                                                  const int32_t *pack_rotations, int32_t pack_rotation_count,
                                                  int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint8_t *out,
                                                  int64_t out_capacity, int64_t *out_count);

/* ---- PNNS in the reference's protobuf messages (pnns_proto.hpp, pnns_plan.hpp) ----
 * Requests as the reference's clients send them and shard responses as they expect them: api.pnns.v1.PNNSRequest and
 * api.pnns.v1.PNNSShardResponse (api/pnns/v1/pnns.proto), their matrices pnns.v1.SerializedCiphertextMatrix
 * (PnnsConversion.swift:265-348, PnnsConversionApi.swift).  The walks refuse what the PIR walks refuse (groups, varints
 * over 10 bytes, lengths past their message, a singular message given twice, a known field of the wrong wire type).
 *
 * hecuda_pnns_request_fields_read: the walk of a PNNSRequest (host only, nothing copied): the number of query matrices
 * and their common num_rows (refused when they differ), the byte ranges (offsets into `bytes`) of config_id, of
 * evaluation_key.evaluation_key (a SerializedEvaluationKey, ready for hecuda_evk_create_proto_many) and of the key
 * identifier, the key timestamp (from evaluation_key_metadata, or evaluation_key.metadata when that is absent), the shard
 * indices and each shard id's (offset, length).  shard_indices / shard_id_ranges (2 x count) may be NULL; otherwise
 * their capacity must hold every entry.  Routing and key caching stay the caller's. */
typedef struct hecuda_pnns_request_fields {
    int32_t query_count;
    uint32_t query_row_count;
    int32_t has_evaluation_key, has_key_metadata;
    int64_t shard_index_count, shard_id_count;
    uint64_t config_id_offset, config_id_bytes;
    uint64_t evaluation_key_offset, evaluation_key_bytes;
    uint64_t key_timestamp, key_identifier_offset, key_identifier_bytes;
} hecuda_pnns_request_fields;
int32_t hecuda_pnns_request_fields_read(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_request_fields *fields,
                                        uint32_t *shard_indices, int64_t index_capacity, uint64_t *shard_id_ranges,
                                        int64_t id_capacity);

/* The size of one client's PNNSShardResponse (Response.proto(), as SwiftProtobuf writes it) for a query of
 * query_row_count rows against matrices[k] on ctxs[k]: per context one .denseColumn SerializedCiphertextMatrix of
 * database rows x query rows whose ciphertexts are SerializedCiphertext.full with that context's
 * Bfv.skipLSBsForDecryption (it depends on t), then entry_ids (packed) and every entry_metadatas element (metadata k is
 * metadata[metadata_offsets[k], metadata_offsets[k + 1])). */
int32_t hecuda_pnns_shard_response_byte_count(const hecuda_context *const *ctxs, int32_t count,
                                              const hecuda_pnns_matrix *const *matrices, int32_t query_row_count,
                                              const uint64_t *entry_ids, int64_t id_count, const uint8_t *metadata,
                                              const uint64_t *metadata_offsets, int64_t metadata_count, uint64_t *bytes);

/* Server.computeResponse for client_count clients, one PNNSRequest per client in (message c: message_byte_counts[c]
 * bytes; only its query matrices are read) and one PNNSShardResponse per client out: out holds client_count x
 * hecuda_pnns_shard_response_byte_count bytes and client c's slice is a complete message.  For every context its reply
 * poly bytes equal what hecuda_pnns_compute_response_clients_wire returns for the same poly0 and seeds.
 *
 * Each request holds one .denseRow matrix per context (wrongCiphertextMatrixCount; wrongMatrixPacking, or unsetOneof
 * for no packing), of the database's column count (invalidMatrixDimensions) and CiphertextMatrix.ciphertextCount(N,
 * dims) ciphertexts (wrongCiphertextCount), every matrix of a request and of every client with client 0's row count.
 * Query ciphertexts may be .seeded or .full (correction factor 1).  The query plan -- each row's ciphertext, mask and
 * replication count, the packing rotations -- is derived here (pnns_plan.hpp) from the shape and client 0's Galois
 * elements, once per call; the masks are SIMD-encoded once per context.
 *
 * evks[c] may belong to any context with the N, word size and coefficient moduli of every ctxs[k] (BFV keys do not
 * depend on t): keys loaded once on ctxs[0] serve every plaintext modulus, read in place, with no copy.  Every Galois
 * key every context's plan needs is found for every client before anything is enqueued; every failure's message starts
 * with "client <c>: " where a client is at fault, and leaves `out` untouched.
 *
 * Per group of HECUDA_PNNS_CLIENT_GROUP clients: one upload of the group's messages; per context the seeded expansion
 * reading poly0 and seeds in place, the many-clients response pipeline and one packing launch per reply poly writing
 * into the clients' messages; one framing launch; one download. */
int32_t hecuda_pnns_compute_response_clients_proto(const hecuda_context *const *ctxs, int32_t count,
                                                   const hecuda_evk *const *evks, int32_t client_count,
                                                   const hecuda_pnns_matrix *const *matrices,
                                                   const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                   const uint64_t *entry_ids, int64_t id_count, const uint8_t *metadata,
                                                   const uint64_t *metadata_offsets, int64_t metadata_count, uint8_t *out);

/* Client side, host only.  hecuda_pnns_request_write: Query.proto() as a PNNSRequest: one .denseRow matrix of
 * row_count x column_count per context k of ciphertext_count .seeded ciphertexts (poly0[k]: ciphertext_count x
 * byteCount(L rows), seeds[k]: ciphertext_count x 32), then config_id when config_id_bytes > 0, then, when
 * evaluation_key is not NULL, evaluation_key { metadata { key_timestamp, key_identifier }, evaluation_key } (a
 * SerializedEvaluationKey).  With out NULL only *written is set; else capacity must hold it.
 * hecuda_pnns_shard_response_read: the walk of a PNNSShardResponse against ctxs (one .denseColumn matrix per context of
 * .full ciphertexts over one modulus, every matrix of one shape): *shape, then, for the arrays that are not NULL,
 * poly_offsets[k x reply_count + r] (offset of reply r's poly 0 in matrix k; poly 1 follows it), skip_lsbs[2k + p],
 * entry_ids[id_count] and metadata_ranges[2 x metadata_count] (offset, length). */
int32_t hecuda_pnns_request_write(const hecuda_context *const *ctxs, int32_t count, uint32_t row_count, uint32_t column_count,
                                  const uint8_t *const *poly0, const uint8_t *const *seeds, int32_t ciphertext_count,
                                  const uint8_t *config_id, uint64_t config_id_bytes, const uint8_t *evaluation_key,
                                  uint64_t evaluation_key_bytes, uint64_t key_timestamp, const uint8_t *key_identifier,
                                  uint64_t key_identifier_bytes, uint8_t *out, uint64_t capacity, uint64_t *written);
typedef struct hecuda_pnns_shard_response_shape {
    int32_t matrix_count, reply_count;
    uint32_t row_count, column_count;
    int64_t id_count, metadata_count;
} hecuda_pnns_shard_response_shape;
int32_t hecuda_pnns_shard_response_read(const hecuda_context *const *ctxs, int32_t count, const uint8_t *bytes,
                                        uint64_t byte_count, hecuda_pnns_shard_response_shape *shape, uint64_t *poly_offsets,
                                        int32_t *skip_lsbs, uint64_t *entry_ids, uint64_t *metadata_ranges);

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
/* scalars: a HOST array of row_count values, scalars[r] < the modulus of row r (read when the call is made), also for
 * the _device variant; only data is a device buffer. */
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

/* ---- client side: secret keys, encryption, evaluation keys, noise budgets (uint64_t only) ----
 * Every random polynomial comes from a NistAes128Ctr(seed:) stream (the generator of hecuda_poly_random_from_seed), one
 * stream per polynomial, keyed by a 32-byte seed the caller supplies.  The reference draws `a` the same way and the
 * secret and the error from SystemRandomNumberGenerator (Bfv+Keys.swift:20-26, Bfv+Encrypt.swift:150-181); here their
 * seeds must come from a cryptographically secure source (the Python layer uses secrets.token_bytes) and must never be
 * reused or revealed.  Each stream maps to coefficients byte for byte as the reference maps its generator:
 *   secret  PolyRq.randomizeTernary (PolyRq+Randomize.swift:87-104): coefficient j takes a little-endian UInt64 and a
 *           UInt32 (stream bytes 12j..12j+11), (u64 << 32 | u32) mod 3, minus 1 modulo every q_i;
 *   error   randomizeCenteredBinomialDistribution (:120-160) at ErrorStdDev.stdDev32 (sigma = 3.2, k = 21): coefficient j
 *           takes two little-endian UInt64 (bytes 16j..16j+15), each masked to k bits, popcount(first) - popcount(second);
 *   a       PolyRq.random (:49-81), sampled in Eval format as hecuda_poly_random_from_seed.
 * Device copies of the secret key, s^2, s(X^g), the errors and the error seeds are zeroized before they are freed.
 *
 * hecuda_bfv_generate_secret_key = Bfv.generateSecretKey (Bfv+Keys.swift:20-26): seeds count x 32 -> secret_keys count x
 * K x N, SecretKey.poly in Eval format over all K coefficient moduli (K = L + 1, or 1 for a single modulus).
 * hecuda_bfv_encrypt = Bfv.encrypt (Bfv+Encrypt.swift:64-72: encryptZero :141-181, then plaintextTranslate(.Add)
 * :75-139) at the top level: secret_key K x N (Eval); plaintexts batch x N Coeff values < t; a_seeds, error_seeds batch x
 * 32 -> ciphertexts batch x 2 x L x N (Coeff) = (-(INTT(a s) + e) + Delta m + adjust, INTT(a)).  A value >= t:
 * HECUDA_ERR_INVALID_ARGUMENT.
 * hecuda_bfv_encrypt_seeded: the same ciphertexts in the .seeded(poly0:seed:) wire form (SerializedCiphertext.swift:41-60):
 * poly0 batch x hecuda_poly_serialized_byte_count(ctx, HECUDA_BASE_Q, L, 0) bytes; the seed is a_seeds[i].  This is what
 * hecuda_ciphertext_expand_seeded and the _clients_wire calls read.
 * hecuda_evk_generate = Bfv.generateEvaluationKey (Bfv+Keys.swift:30-65, _generateKeySwitchKey :67-103): for each key,
 * key ciphertext i is encryptZero over [q_0..q_{L-1}, q_ks] in Eval with (q_ks mod q_i) currentKey[i] added to row i of
 * poly0; currentKey = s^2 for the relinearization key (has_relin != 0), s(X^g) for each element g (Galois.swift:151-166).
 * a_seeds and error_seeds: (has_relin + element_count) x L x 32 bytes, in hecuda_evk_create_serialized's order (the
 * relinearization key, then elements[]).  *out is an ordinary evaluation key.  wire_poly0 (nullable): the keys' poly0 in
 * hecuda_evk_create_serialized's layout, so that (wire_poly0, a_seeds) loads the same key there.  Errors as
 * hecuda_evk_create_serialized, plus HECUDA_ERR_MISSING_KEY for a null secret key and HECUDA_ERR_INVALID_ARGUMENT for null
 * seeds; on error *out is NULL and nothing was launched.
 * hecuda_bfv_noise_budget = Bfv.noiseBudgetEval / noiseBudgetCoeff (Bfv+Decrypt.swift:116-185): ciphertexts batch x
 * poly_count x moduli_count x N (Coeff, or Eval with eval_format != 0; poly_count 2 or 3, any level) -> budgets[batch] =
 * log2(qDouble / (2 norm)), norm = the largest centred |[t (c0 + c1 s (+ c2 s^2))]_q| as a Double (round to nearest),
 * qDouble the running product of Double(q_i); +inf for a zero norm.
 * WARNING (Bfv+Decrypt.swift:111-112): a noise budget must never be forwarded to any other party.  Sharing it acts as an
 * oracle that can be used to recover the secret key. */
int32_t hecuda_bfv_generate_secret_key(const hecuda_context *ctx, const uint8_t *seeds, uint64_t *secret_keys, int64_t count);
int32_t hecuda_bfv_encrypt(const hecuda_context *ctx, const uint64_t *secret_key, const uint64_t *plaintexts,
                           const uint8_t *a_seeds, const uint8_t *error_seeds, uint64_t *ciphertexts, int64_t batch);
int32_t hecuda_bfv_encrypt_seeded(const hecuda_context *ctx, const uint64_t *secret_key, const uint64_t *plaintexts,
                                  const uint8_t *a_seeds, const uint8_t *error_seeds, uint8_t *poly0, int64_t batch);
int32_t hecuda_evk_generate(const hecuda_context *ctx, const uint64_t *secret_key, int32_t has_relin, const uint32_t *elements,
                            int32_t element_count, const uint8_t *a_seeds, const uint8_t *error_seeds, hecuda_evk **out,
                            uint8_t *wire_poly0);
int32_t hecuda_bfv_noise_budget(const hecuda_context *ctx, const uint64_t *secret_key, const uint64_t *ciphertexts,
                                int32_t poly_count, int32_t moduli_count, int32_t eval_format, double *budgets, int64_t batch);

/* hecuda_evk_copy: a device-to-device copy of `evk` (its relinearization key and every Galois key) owned by `ctx`, as
 * the reference uses one evaluation key generated on contexts[0] with every plaintext modulus (PrivateNearestNeighborSearch/
 * Client.swift:137-146: BFV keys do not depend on t).  Refused (HECUDA_ERR_INVALID_ARGUMENT) unless N, the word size
 * and the coefficient moduli, in order and including the key-switching modulus, are identical.  The copy is
 * independent of `evk` (either may be destroyed first).  On error *out is NULL and nothing is launched. */
int32_t hecuda_evk_copy(const hecuda_evk *evk, const hecuda_context *ctx, hecuda_evk **out);

/* ---- PNNS client and float database processing (uint64_t only) ----
 * Array2d.normalizedScaledAndRounded (PrivateNearestNeighborSearch/Util.swift:74-89) in Swift Float arithmetic: per
 * row, the squares summed left to right in float32, a correctly rounded square root, then for each value
 * (value * Float(scaling_factor)) / norm rounded twice and .toNearestOrAwayFromZero into Int64; a zero-norm row is 0.
 * Every operation is rounded on its own (no FMA contraction).  Where Swift traps -- a non-finite input, a value outside
 * Int64, or (without reduce) outside [-floor(t/2), floor((t-1)/2)] -- the call returns HECUDA_ERR_INVALID_ARGUMENT.
 *
 * hecuda_pnns_matrices_create_from_vectors = Database.process (ProcessedDatabase.swift:194-229) for the .diagonal
 * packing: vectors row_count x column_count floats, row-major; one matrix per context (ctxs[0 .. plaintext_count), all
 * with the same N), each the handle hecuda_pnns_matrix_create_from_values builds from the normalised values with
 * reduce = (plaintext_count > 1) (:213-214).  The floats cross PCIe once and are normalised once.  On error every out[k]
 * is NULL and nothing stays allocated.
 *
 * hecuda_pnns_query_generate = Client.generateQuery for one context (Client.swift:73-91): normalise, pack .denseRow
 * (PlaintextMatrix.swift:341-413) into ceil(rows / (N / nextPow2(cols))) SIMD plaintexts, encode, encrypt
 * (hecuda_bfv_encrypt: secret_key K x N Eval, a_seeds / error_seeds one 32-byte seed per ciphertext), all on the device.
 * reduce: Modulus.reduce instead of centeredToRemainder (the reference reduces when there are several plaintext
 * moduli).  Exactly one of ciphertexts (count x 2 x L x N, Coeff) and poly0 (count x byteCount(L rows), the
 * .seeded(poly0:seed: a_seeds[i]) wire form) is non-null.  A non-finite input, column_count outside 1 .. N/2, or a
 * scaling factor whose values cannot fit the plaintext map is refused before anything is launched.
 *
 * hecuda_pnns_decrypt_distances = Client.decrypt (Client.swift:99-127): replies[k] is the .denseColumn response matrix of
 * context k (reply_count x 2 x moduli_count x N, Coeff; reply_count as the reference packs matrix_rows x query_rows
 * values).  Per context: the decryption dot product and scale-and-round (hecuda_bfv_decrypt), SIMD decode; then one
 * kernel: unpackDenseColumn (PlaintextMatrix.swift:515-555), CrtComposer.compose (CrtComposer.swift:76-97),
 * remainderToCentered over prod t and Float(signed) / (Float(s) * Float(s)).  distances: matrix_rows x query_rows float,
 * row-major (MatrixMultiplication.swift:291-293).  The contexts must differ only in t; refused: 2 prod t above UInt64.max
 * with several moduli (composeMaxIntermediateValue), plaintext moduli that are not pairwise distinct, more than 8
 * contexts.  The device copy of the secret key is zeroized before it is freed. */
int32_t hecuda_pnns_matrices_create_from_vectors(const hecuda_context *const *ctxs, int32_t plaintext_count, const float *vectors,
                                                 int64_t row_count, int64_t column_count, int64_t scaling_factor,
                                                 int32_t baby_step, int32_t giant_step, hecuda_pnns_matrix **out);
int32_t hecuda_pnns_query_generate(const hecuda_context *ctx, const uint64_t *secret_key, const float *vectors, int64_t row_count,
                                   int64_t column_count, int64_t scaling_factor, int32_t reduce, const uint8_t *a_seeds,
                                   const uint8_t *error_seeds, uint64_t *ciphertexts, uint8_t *poly0);
int32_t hecuda_pnns_decrypt_distances(const hecuda_context *const *ctxs, int32_t plaintext_count, const uint64_t *secret_key,
                                      const uint64_t *const *replies, int64_t reply_count, int32_t moduli_count,
                                      int64_t matrix_rows, int64_t query_rows, int64_t scaling_factor, float *distances);

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
