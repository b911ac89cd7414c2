// context.hpp -- immutable device context: moduli, NTT root tables and BEHZ / key-switch constants.
//
// Host-side construction mirrors what the reference precomputes in Context<Bfv<UInt64>>.init
// (Sources/HomomorphicEncryption/Context.swift:94-143), PolyContext.init (PolyRq/PolyContext.swift:45-123),
// _NttContext.init (PolyRq/PolyRq+Ntt.swift:118-169) and _RnsTool.init (RnsTool.swift:132-251).
// Where the reference applies two exact modular steps in a row, the constants here are pre-multiplied so the
// kernels do one multiply-accumulate pass (see DESIGN.md "fused constants"); results are the same canonical residues.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "modarith.cuh"

namespace hecuda {

constexpr int kMaxL = 32;               // coefficient moduli: the reference allows 32 (EncryptionParameters.swift:148)
constexpr int kMaxSlots = 3 * kMaxL + 4;  // q_0..q_{L-1} | bsk_0..bsk_L | q_ks | aux_0..aux_L | t
constexpr int kMaxRows = 2 * kMaxL + 1;

// One NTT-capable modulus.  Twiddle tables are interleaved (w, floor(w 2^64 / p)) pairs, indexed like the
// reference's rootOfUnityPowers: entry m + i serves group i of the stage with m groups (PolyRq+Ntt.swift:128-137).
struct ModSlot {
    u64 p;
    u64 mu1;          // floor(2^64 / p)
    u64 mu_hi, mu_lo; // floor(2^128 / p)
    u64 mu_prod;      // floor(2^(bits+62) / p)
    int s_prod;       // bits - 2
    int bits;
    int red_shift;    // max(bits - 12, 0)             } small-quotient reduction of lazy NTT values (< 512 p),
    u32 red_recip;    // floor(2^(red_shift+32) / p)   } ntt_fast.cuh::reduce_small
    u64 ninv;         // -p^-1 mod 2^64 (Montgomery)
    u64 r64;          // 2^64 mod p
    // Last inverse-NTT stage: x' = (x + y) c0, y' = (x - y) c1 with c0 = s N^-1, c1 = s N^-1 psi^-(N/2)
    // (PolyRq+Ntt.swift:159-168,416-419) for three scalings s:
    //   kScalePlain  s = 1                 the reference's inverseNtt
    //   kScaleTMont  s = t 2^64            after the Montgomery-form tensor product; folds `poly * tVec` (Bfv+Multiply.swift:40)
    //   kScaleMont   s = 2^64              after the Montgomery-reduced key-switch accumulation
    //   kScaleTMontFloor  s = t 2^64 (Q/q_i)^-1 on the ciphertext moduli q_i, t 2^64 elsewhere: kScaleTMont with the
    //                     floor's first step y_i = [x_i (Q/q_i)^-1]_{q_i} (RnsTool.swift:378-398) folded in
    struct InvScale { u64 c0, c0p, c1, c1p; } inv_scale[4];
    const ulonglong2 *tw;     // forward twiddles  [N]
    const ulonglong2 *itw;    // inverse twiddles  [N]  (itw[m+i] = tw[m+i]^-1)
    // transposed copies for the register-tiled kernels' line-owning pass (ntt_fast.cuh): entry k (< 15) of thread
    // tau (< N/16) at [k * N/16 + tau]; null when N is outside the fast kernels' range or has the resident image
    const ulonglong2 *tw_t;
    const ulonglong2 *itw_t;
    // N = 2^13: every twiddle the fast kernels read, laid out as a CTA keeps them in shared memory (ntt_fast.cuh,
    // resident_twiddles); null at other sizes
    const ulonglong2 *tw_img;
    const ulonglong2 *itw_img;
};

enum { kScalePlain = 0, kScaleTMont = 1, kScaleMont = 2, kScaleTMontFloor = 3 };

struct NttRowMap {       // which modulus slot each row of a polynomial uses:
    int rows_per_poly;   //   slot[((row % rows_per_poly) / group)]
    int group;
    unsigned char slot[kMaxRows + 1];
    // Optional gather on the input side (forward NTT only), used for key-switch digits (Bfv+Keys.swift:165-179):
    // output row idx of polynomial k reads source row (idx % src_mod) at in + k * src_poly_stride, whose residues are
    // mod the modulus in slot src_slot[idx % src_mod] and are re-reduced into the row's modulus where needed.
    int src_mod;                  // 0 = no gather (input laid out like the output)
    long long src_poly_stride;    // words
    unsigned char src_slot[kMaxRows + 1];
};

// liftQToQBsk (RnsTool.swift:324-368) fused to: z_i = [x_i * in_w_i]_{q_i} (canonical);
//   r = [ -Q^-1 * sum_i z_i (Q/q_i) ]_{2^32}, centered;
//   out_j = [ (sum_i z_i mat[j][i] + r_c qr[j]) 2^-64 ]_{b_j}   with mat, qr pre-multiplied by 2^64 (Montgomery)
struct LiftConsts {
    int L;
    int wide_sums;                   // the lazy sums may exceed 2 b_j: finish with a Barrett reduction (many wide moduli)
    u64 b_mu1[kMaxL + 1];            // floor(2^64 / b_j)
    u64 q[kMaxL];
    u64 in_w[kMaxL], in_wp[kMaxL];   // m~ (Q/q_i)^-1 mod q_i
    u32 punct_mt[kMaxL];             // (Q/q_i) mod m~
    u32 neg_inv_q_mt;                // -Q^-1 mod m~
    u32 mt_mask, mt_half;            // m~ - 1, m~ / 2   (m~ = 2^32 for Bfv<UInt64>, 2^16 for Bfv<UInt32>, Scalar.swift:498-525)
    u64 neg_off[kMaxL + 1];          // k b_j - m~ >= 0 with the least such k: the centered r - m~ as a residue mod b_j
    u64 b[kMaxL + 1], b_ninv[kMaxL + 1];
    u64 mat[kMaxL + 1][kMaxL];       // (Q/q_i) m~^-1 2^64 mod b_j
    u64 qr[kMaxL + 1];               // Q m~^-1 2^64 mod b_j
    int h_primes;                    // every b_j is h 2^32 + 1 < 2^55: reduce with mont_reduce_h
};

// floorQBskToQ (RnsTool.swift:378-456) fused to (all matrix constants pre-multiplied by 2^64, sums Montgomery-reduced):
//   y_i = [x_i inq_w_i]_{q_i} (canonical);  f_j = [x_bj fq[j] + sum_i y_i fmat[j][i]]_{b_j}  (approximateFloor)
//   for j = k < L the row constants also carry (B/b_k)^-1, so f_k is already w_k = [f_k (B/b_k)^-1]_{b_k} (canonical
//   after a conditional subtraction, or a Barrett reduction with wide_sums);  f_msk = f_L stays lazy (< 2 m_sk)
//   alpha = [sum_k w_k amat[k] + f_msk a_msk]_{m_sk}  (Shenoy-Kumaresan)
//   out_i = [sum_k w_k omat[i][k] + alpha' D_i]_{q_i},  (alpha', D) = alpha > m_sk/2 ? (m_sk-alpha, B) : (alpha, -B)
struct FloorConsts {
    int L;
    int wide_sums;                     // alpha may exceed 8 m_sk: finish with a Barrett reduction
    u64 msk_mu1;                       // floor(2^64 / m_sk)
    u64 q[kMaxL], q_ninv[kMaxL], q_mu1[kMaxL];
    u64 inq_w[kMaxL], inq_wp[kMaxL];   // (Q/q_i)^-1 mod q_i
    u64 b[kMaxL + 1], b_ninv[kMaxL + 1];
    u64 b_mu1[kMaxL + 1];              // floor(2^64 / b_j)
    u64 fq[kMaxL + 1];                 // Q^-1 2^64 [(B/b_j)^-1 for j < L] mod b_j
    u64 fmat[kMaxL + 1][kMaxL];        // -(Q/q_i) Q^-1 2^64 [(B/b_j)^-1 for j < L] mod b_j
    u64 amat[kMaxL];                   // (B/b_k) B^-1 2^64 mod m_sk
    u64 a_msk;                         // -B^-1 2^64 mod m_sk
    u64 omat[kMaxL][kMaxL];            // (B/b_k) 2^64 mod q_i
    u64 b_mod_q[kMaxL], neg_b_mod_q[kMaxL];  // +-B 2^64 mod q_i
    int h_primes;                      // every b_j is h 2^32 + 1 < 2^55: reduce f_j and alpha with mont_reduce_h
};

// divideAndRoundQLast (PolyRq.swift:365-393) for a base [m_0..m_{l-2}, m_last]
struct DivRoundConsts {
    int l;                              // rows in (including the last)
    u64 m[kMaxL + 1], mu1[kMaxL + 1];   // moduli of the kept rows + Barrett factor
    u64 last, half;                     // m_last, m_last >> 1
    u64 half_mod[kMaxL + 1];            // half mod m_i
    u64 inv_w[kMaxL + 1], inv_wp[kMaxL + 1];  // m_last^-1 mod m_i
};

// Plaintext translate at level l (Bfv+Encrypt.swift:75-139) over Q_l = q_0..q_{l-1} (getRnsTool(moduliCount: l)):
//   adjust = floor(([Q_l]_t m + tThreshold) / t),   c0_i +-= [floor(Q_l / t) m + adjust]_{q_i}
// [Q_l]_t m + tThreshold < t^2 may exceed 64 bits (t up to 2^62): with w = [Q_l]_t and r = [w m]_t,
// floor((w m + tThreshold) / t) = floor(w m / t) + (r + tThreshold >= t), and floor(w m / t) is the quotient of the
// Shoup multiplication by w modulo t (wp = floor(w 2^64 / t)) -- exact without a 128-bit division.
struct TranslateConsts {
    int l;
    u64 t, t_threshold;                  // t, (t + 1) / 2   (RnsTool.tThreshold, RnsTool.swift:123-125)
    u64 q_mod_t, q_mod_t_p;              // [Q_l]_t and its Shoup factor modulo t   (RnsTool.qModT, :167)
    u64 q[kMaxL];
    u64 delta[kMaxL], delta_p[kMaxL];    // floor(Q_l / t) mod q_i and Shoup factors (RnsTool.qDivT, :176-182)
};

struct HostSlot {
    ModSlot dev;                      // with device pointers filled in
    std::vector<u64> roots, inv_roots;  // host copies (w only) for parity checks
};

class Context {
   public:
    // word_bits: the reference's scalar type -- 64 = Bfv<UInt64>, 32 = Bfv<UInt32> (its m~, gamma and Bsk, moduli < 2^30)
    static Context *create(int64_t n, const u64 *coeff_moduli, int nmod, u64 t, std::string &err, int word_bits = 64);
    ~Context();

    int64_t n;
    int logn;
    int word_bits = 64;
    u64 mtilde = 1ull << 32;   // T.mTilde
    u64 gamma = (1ull << 62) - 40797;  // T.rnsCorrectionFactor
    int L;           // ciphertext moduli
    u64 t;
    int device;
    int sm_count;
    std::vector<u64> q;    // q_0..q_{L-1}
    u64 q_ks;              // 0 when the parameters have a single coefficient modulus: no key-switching modulus, no
    bool has_ks = true;    // evaluation keys (Context.swift:102-107, supportsEvaluationKey == false)
    std::vector<u64> bsk;  // L+1 primes: the reference's BEHZ base (RnsTool.swift:30-33)
    std::vector<u64> aux;  // L+1 primes: the base ct x ct multiply actually computes in (context.cu); == bsk when
    bool aux_is_reference = true;  // the conditions for the faster base do not hold (or HECUDA_AUX_BASE=reference)
    // the most tensor products one floor may sum over aux (ct x ct inner product); larger sums run over Bsk
    int64_t aux_max_pairs = INT64_MAX;
    std::vector<HostSlot> slots;  // L q's, L+1 bsk, 1 q_ks, then L+1 aux (when different from bsk), then t (SIMD)
    ModSlot *d_slots = nullptr;   // device array: the slots, then (N = 2^15 only) 2 virtual half-transform slots per slot
    int split_slot_base = 0;      // index of the first virtual slot (slot s, half h -> split_slot_base + 2 s + h)
    LiftConsts lift;        // over [Q, Bsk]: stage-level entry points
    FloorConsts floor;
    LiftConsts lift_mul;    // over [Q, aux]: Bfv.mulAssign / innerProduct
    FloorConsts floor_mul;
    std::vector<DivRoundConsts> ks_divround;   // index l (1..L): base [q_0..q_{l-1}, q_ks]
    std::vector<DivRoundConsts> ms_divround;   // index l (2..L): base [q_0..q_{l-1}]
    void *d_pool = nullptr;  // twiddle storage
    // SIMD encoding (Encoding.swift:197-245): present when t is a prime = 1 mod 2N (isNttModulus, PolyRq+Ntt.swift:24-27)
    bool simd = false;
    int32_t *d_simd_matrix = nullptr;  // [N] generateEncodingMatrix: slot i <-> Eval position matrix[i]
    int32_t *d_simd_inverse = nullptr; // [N] inverse permutation: Eval position j holds slot inverse[j]
    std::vector<TranslateConsts> translate;  // index l (1..L)

    int slot_q(int i) const { return i; }
    int slot_bsk(int j) const { return L + j; }
    int slot_ks() const { return 2 * L + 1; }
    int slot_aux(int j) const { return aux_is_reference ? slot_bsk(j) : 2 * L + 2 + j; }
    // the plaintext modulus, after every other slot (Context.plaintextContext); -1 without SIMD support
    int slot_t() const { return simd ? (aux_is_reference ? 2 * L + 2 : 3 * L + 3) : -1; }
    NttRowMap map_q(int rows) const;      // rows of the ciphertext context
    NttRowMap map_qbsk() const;           // [Q, Bsk]
    NttRowMap map_qaux() const;           // [Q, aux]
    NttRowMap map_ks(int l) const;        // [q_0..q_{l-1}, q_ks]
    NttRowMap map_single(int slot) const;
    // (l+1) x l digit rows, row (r, j) = [target row j]_{m_r}; gathered from target polynomials `stride` words apart
    NttRowMap map_ks_digits(int l, long long target_poly_stride) const;
    int find_slot(u64 modulus) const;
};

}  // namespace hecuda
