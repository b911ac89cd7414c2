// ntt_fast.cuh -- register-tiled negacyclic NTT passes over a row staged in shared memory (shared by the sm_90a
// kernels in ntt_fast.cu and by the host-side SIMT emulation in tests/emu/ntt_emulate.cu, which replays the exact
// index maps and lazy-reduction schedule on the CPU).
//
// One team of T = N/16 threads transforms one row of N = 2^LOGN residues.  The row lives in shared memory for the
// whole transform (it arrives and leaves by TMA bulk copies, one 128-byte line per thread, see ntt_fast.cu); every
// thread keeps 16 residues in registers and runs up to 4 butterfly stages on them between two shared-memory exchanges.
//
// A pass (LB, C) covers the C consecutive stages whose butterfly partners differ in element-index bits [LB, LB + C).
// A thread's 16 registers hold the 2^C values of those bits times 2^E "passenger" values of the low bits [0, E),
// E = 4 - C (no passengers when LB == 0, where C == 4):
//     e = (hi << (LB + C)) | (a << LB) | (lo << E) | f,    a < 2^C, f < 2^E,   register r = (a << E) | f
//     lo = tau & (2^(LB-E) - 1),  hi = tau >> (LB - E)
// so whenever E >= 1 (or LB == 0) registers 2k, 2k+1 are adjacent residues: every shared-memory access is 128-bit.
// Passengers sit below the stage bits, hence all of a thread's butterflies of one stage group share a twiddle:
//   forward (Cooley-Tukey, reference _NttContext.forwardNtt, PolyRq+Ntt.swift:237-319): stages s = S0 + j
//       (S0 = LOGN - LB - C), pair distance 2^(C-1-j) in `a`, twiddle index 2^s + (hi << j) + (a >> (C-j))
//   inverse (Gentleman-Sande, PolyRq+Ntt.swift:379-483): pair distance 2^j in `a`, m = 2^(LOGN-1-LB-j) groups,
//       twiddle index m + (hi << (C-1-j)) + (a >> (j+1)); the stage with m = 1 multiplies by N^-1 and
//       N^-1 psi^-(N/2) (optionally times t or 2^64).
// The LB == 0 pass (last forward / first inverse) gives every thread its own 15 twiddles; they come from a transposed
// copy of the table (entry k of thread tau at [k * T + tau]) so each load instruction of a warp is one contiguous
// 512-byte request.  At N = 2^13 that copy lives in shared memory with the rest of the twiddles (the resident image,
// see resident_twiddles below); the other sizes read it from global memory.
//
// Shared-memory layout: the TMA unit's 128-byte swizzle (CU_TENSOR_MAP_SWIZZLE_128B) -- the 16-byte chunk c of the
// 128-byte line r is stored at chunk c ^ (r & 7), i.e. word index phys(e) = e ^ (((e >> 4) & 7) << 1).  The row needs
// no padding (exactly N words) and one bulk-tensor copy moves 256 lines.  phys is XOR-linear over disjoint bit
// fields: phys(base | field) = phys(base) ^ phys(field), and whenever the field stays clear of element bits 1..6 the
// XOR is an addition, so accesses are (per-thread base) + (compile-time offset); the two passes whose register bits
// reach into bits 1..6 spend one LOP3 per 128-bit access.  All passes of all plans are bank-conflict free in this
// layout (tests/test_ntt_emulation.py checks it).
//
// Modular arithmetic.  The Shoup product uses an under-estimated quotient q~ = y1 w'1 + hi(y1 w'0) + hi(y0 w'1)
// (3 wide multiplies instead of 4 + carries; never above floor(y w'/2^64), at most 2 below), so products land in
// [0, 4p).  What the reference fixes is the canonical residue written back (PolyRq.swift:36), not the lazy ranges:
//   NARROW (p < 2^55): forward never reduces (values < (2 + 4 LOGN) p), inverse lets values double per stage and
//       reduces once at the entry of the pass that could overflow; both finish with a one-multiply small-quotient
//       reduction.
//   MID (p < 2^61): Harvey-style with doubled ranges, [0, 8p) forward (one conditional subtraction of 4p per
//       butterfly), [0, 4p) inverse.
//   WIDE (p < 2^62): exact quotient, [0, 4p) forward / [0, 2p) inverse (the reference's own ranges).
//   NARROW-H (p = h 2^32 + 1 < 2^55): NARROW's ranges; the product q~ p needs one 32-bit multiply (q~0 h) instead of a
//       wide one plus two: 4 IMAD.WIDE + 3 IMAD per butterfly.
//   SMALL (p < 2^30, the moduli of the reference's Bfv<UInt32> and of the default PIR parameters): the butterflies
//       run in 32-bit arithmetic -- one IMAD.HI and two IMAD per Shoup product instead of five IMAD.WIDE and four IMAD --
//       on Harvey's ranges, with the 32-bit Shoup factor taken from the top half of the 64-bit one
//       (floor(floor(w 2^64 / p) / 2^32) = floor(w 2^32 / p)); residues stay zero-extended in their 64-bit slots.
#pragma once
#include "context.hpp"
#include "modarith.cuh"

namespace hecuda {
namespace fast {

constexpr int kMinLogN = 10, kMaxLogN = 14;
constexpr int kSplitLogN = 15;  // one cross-half stage in global memory + two kMaxLogN transforms (ntt_fast.cu)
constexpr int kNarrowBits = 55;  // reduction-free butterflies: lazy values < 512 p < 2^64
constexpr int kMidBits = 61;     // 8 p < 2^64
constexpr int kSmallBits = 30;   // Modulus<UInt32>.max = 2^30 - 1: the reference's 32-bit word size (Modulus.swift:177-180)
enum { kNarrow = 0, kMid = 1, kWide = 2, kSmall = 3, kNarrowH = 4 };
HE_HD constexpr int class_of_bits(int bits) {
    return bits <= kSmallBits ? kSmall : bits <= kNarrowBits ? kNarrow : bits <= kMidBits ? kMid : kWide;
}
// NARROW primes of the form h 2^32 + 1 (the auxiliary primes context.cu picks for the multiply): the q p product of a
// Shoup multiplication collapses to q + ((q0 h) << 32)
HE_HD constexpr int class_of_modulus(u64 p, int bits) {
    return (class_of_bits(bits) == kNarrow && (u32)p == 1u) ? kNarrowH : class_of_bits(bits);
}
HE_HD constexpr bool narrow_like(int cls) { return cls == kNarrow || cls == kNarrowH; }

// Class sets: the instruction streams one kernel instantiation carries (ntt_fast.cu).  Every class's passes are fully
// unrolled, so each stream costs several thousand instructions of code.  The all-class kernels carry no NARROW-H stream:
// there a NARROW-H row runs NARROW's butterflies, which are valid for every p < 2^55.  The N = 2^13 multiply's rows
// ([Q, aux] with 55-bit q_i and h 2^32 + 1 auxiliary primes) get a kernel with just the two streams they use.
HE_HD constexpr unsigned class_bit(int cls) { return 1u << cls; }
constexpr unsigned kAllClasses = (1u << kNarrow) | (1u << kMid) | (1u << kWide) | (1u << kSmall);
constexpr unsigned kNarrowClasses = (1u << kNarrow) | (1u << kNarrowH);
HE_HD constexpr bool has_class(unsigned set, int cls) { return (set & class_bit(cls)) != 0; }

// ---- pass plans: stage counts of the forward passes, in execution order; the inverse runs the mirrored list
HE_HD constexpr int plan_passes(int logn) { return logn <= 12 ? 3 : 4; }
HE_HD constexpr int plan_c(int logn, int k) {
    return logn == 10   ? (k == 2 ? 4 : 3)
           : logn == 11 ? (k == 1 ? 3 : 4)
           : logn == 12 ? 4
           : logn == 13 ? (k == 3 ? 4 : 3)
                        : (k == 0 || k == 3 ? 4 : 3);
}
HE_HD constexpr int fwd_c(int logn, int k) { return plan_c(logn, k); }
HE_HD constexpr int fwd_lb(int logn, int k) {
    int s0 = 0;
    for (int i = 0; i < k; ++i) s0 += plan_c(logn, i);
    return logn - s0 - plan_c(logn, k);
}
HE_HD constexpr int inv_c(int logn, int k) { return plan_c(logn, plan_passes(logn) - 1 - k); }
HE_HD constexpr int inv_lb(int logn, int k) {
    int u0 = 0;
    for (int i = 0; i < k; ++i) u0 += inv_c(logn, i);
    return u0;
}
HE_HD constexpr int pass_e(int lb, int c) { return lb == 0 ? 0 : 4 - c; }  // passenger bits

// NARROW inverse bounds, in units of p.  A stage with inputs < b p outputs x' < 2 b p and y' < 4p, so the bound
// evolves as b -> max(2b, 4), and needs 2 b p < 2^64, i.e. b <= 256 for p < 2^55.
HE_HD constexpr int inv_stage_bound(int b) { return 2 * b > 4 ? 2 * b : 4; }
HE_HD constexpr int inv_bound_after(int b, int stages) {
    for (int i = 0; i < stages; ++i) b = inv_stage_bound(b);
    return b;
}
HE_HD constexpr bool inv_pass_fits(int b, int stages) {  // every stage of the pass sees inputs <= 256 p
    for (int i = 0; i < stages; ++i) {
        if (b > 256) return false;
        b = inv_stage_bound(b);
    }
    return true;
}
// whether pass k reduces its inputs on entry, and the bound on its inputs after that
HE_HD constexpr bool inv_reduce_at(int logn, int k) {
    int b = 1;
    bool red = false;
    for (int i = 0; i <= k; ++i) {
        const int c = inv_c(logn, i);
        red = !inv_pass_fits(b, c);
        if (red) b = 1;
        b = inv_bound_after(b, c);
    }
    return red;
}
HE_HD constexpr int inv_bound_in(int logn, int k) {
    int b = 1;
    for (int i = 0; i <= k; ++i) {
        const int c = inv_c(logn, i);
        if (!inv_pass_fits(b, c)) b = 1;
        if (i < k) b = inv_bound_after(b, c);
    }
    return b;
}

// ---- shared-memory layout
HE_HD constexpr int smem_phys(int e) { return e ^ (((e >> 4) & 7) << 1); }
HE_HD constexpr int smem_words(int logn) { return 1 << logn; }
constexpr int kLineWords = 16;
constexpr int kBoxLines = 256;  // lines moved by one bulk-tensor copy (box = 16 x 256 words = 32 KB)

HE_HD ulonglong2 ld_tw(const ulonglong2 *p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// element index of register r of thread tau in pass (LB, C)
template <int LOGN, int LB, int C>
HE_HD int elem_index(int tau, int r) {
    constexpr int E = pass_e(LB, C);
    const int lo = tau & ((1 << (LB - E)) - 1), hi = tau >> (LB - E);
    return (hi << (LB + C)) | ((r >> E) << LB) | (lo << E) | (r & ((1 << E) - 1));
}
template <int LB, int C>
HE_HD constexpr int reg_offset(int r) {  // compile-time part of the element index
    return ((r >> pass_e(LB, C)) << LB) | (r & ((1 << pass_e(LB, C)) - 1));
}
template <int LB, int C>
HE_HD constexpr bool pass_vec() { return pass_e(LB, C) >= 1 || LB == 0; }

// word index of register r, given the thread's phys(base): an addition when the register field avoids the swizzled bits
template <int LB, int C>
HE_HD int reg_word(int base_phys, int r) {
    constexpr int kSwizzled = 0x7e;  // element bits 1..6 take part in the XOR
    const int off = reg_offset<LB, C>(r);
    return (off & kSwizzled) ? (base_phys ^ smem_phys(off)) : (base_phys + off);
}

template <int LOGN, int LB, int C>
HE_HD void load_smem(u64 (&x)[16], const u64 *sm, int tau) {
    const int b = smem_phys(elem_index<LOGN, LB, C>(tau, 0));
    if (pass_vec<LB, C>()) {
#pragma unroll
        for (int r = 0; r < 16; r += 2) {
            const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(sm + reg_word<LB, C>(b, r));
            x[r] = v.x;
            x[r + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int r = 0; r < 16; ++r) x[r] = sm[reg_word<LB, C>(b, r)];
    }
}
template <int LOGN, int LB, int C>
HE_HD void store_smem(const u64 (&x)[16], u64 *sm, int tau) {
    const int b = smem_phys(elem_index<LOGN, LB, C>(tau, 0));
    if (pass_vec<LB, C>()) {
#pragma unroll
        for (int r = 0; r < 16; r += 2)
            *reinterpret_cast<ulonglong2 *>(sm + reg_word<LB, C>(b, r)) = make_ulonglong2(x[r], x[r + 1]);
    } else {
#pragma unroll
        for (int r = 0; r < 16; ++r) sm[reg_word<LB, C>(b, r)] = x[r];
    }
}

// Per-row constants.  Only what every butterfly needs is held in registers across the row; everything used once
// per row (reduction constants, final-stage scalings) is read from the slot when it is needed.
struct RowMod {
    u64 np;           // 2^64 - p: lets the Shoup product be all multiply-adds (y w + q np)
    u64 kp;           // NARROW / MID: 4p, WIDE: 2p  (the offset that keeps x - v non-negative)
    const ulonglong2 *tw;    // twiddles of this direction, indexed like the reference's rootOfUnityPowers (host emulation)
    unsigned tw_s;           // device: shared-memory address of the CTA's copy of tw[0 .. N/16) (the LB > 0 passes), or
                             // at N = 2^13 of the resident image
    const ModSlot *slot;     // p, mu1, red_shift, red_recip, inv_scale[scale_mode], tw_t / itw_t
    int scale_mode;          // < 0: forward transform
    bool partial;            // inverse only: this row is one half of a 2^15 transform -- its last stage is an ordinary
                             // butterfly (twiddle entry 1 of its table) and the N^-1 scaling happens in the merge kernel
    // transposed copy of the twiddles for the LB == 0 pass: entry k of thread tau at [k * T + tau]
    HE_HD const ulonglong2 *tw_t() const { return scale_mode < 0 ? slot->tw_t : slot->itw_t; }
};

// ---- resident twiddle image (N = 2^13)
// There one CTA runs per SM (ntt_fast.cu) and walks many consecutive rows of one modulus, but the transposed table of
// the LB == 0 pass is 15 x 8 KB = 120 KB, read once per row from L2 -- nearly twice the row itself.  So the CTA keeps
// every twiddle of the transform in shared memory, loaded by one bulk copy when the row's modulus changes:
//     image = [tw[0 .. T): the LB > 0 passes][LB == 0 pass: slot k' (< 11) of thread tau at T + k' T + tau]
// Of the LB == 0 stage with N/2 twiddles (forward stage j = 3, inverse stage J = 0) only the even groups are kept:
// entries i - 1 and i (i odd) of that stage differ in bit 0 of i, i.e. by N/2 in the exponent of psi (the tables are
// bit-reversed), so w_i = w_(i-1) zeta with zeta = psi^(N/2) = tw[1] (inverse: psi^(-N/2) = itw[1]), which is image
// entry 1.  The odd groups multiply their operand by zeta and then by the even group's twiddle.  11 slots a thread
// instead of 15: the image is 8 KB + 11 x 8 KB = 96 KB, and with the two 64 KB row buffers a CTA needs 229 400 bytes of
// the 232 448 it may have (with all 15 slots, 262 168 would not fit).  N <= 2^12 (several CTAs per SM) and N = 2^14
// (one 128 KB row buffer) keep the global transposed table.
HE_HD constexpr bool resident_twiddles(int logn) { return logn == 13; }
constexpr int kImageSlots = 11;
HE_HD constexpr int image_entries(int logn) { return (1 << (logn - 4)) * (1 + kImageSlots); }
// the transposed entry k (< 15, see fwd_last_source / inv_first_source) that image slot k' holds
HE_HD constexpr int fwd_image_k(int kp) { return kp < 7 ? kp : 7 + 2 * (kp - 7); }    // stage j = 3: even groups
HE_HD constexpr int inv_image_k(int kp) { return kp < 4 ? 2 * kp : kp + 4; }          // stage J = 0: even groups

// twiddle `index` (< N/16) of the LB > 0 passes: from the CTA's shared-memory copy on the device
HE_HD ulonglong2 ld_tw_cached(const RowMod &m, int index) {
#if defined(__CUDA_ARCH__)
    ulonglong2 v;
    asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "r"(m.tw_s + (unsigned)index * 16u));
    return v;
#else
    return m.tw[index];
#endif
}
// slot k' of thread tau (< T = N/16) of the resident image: on the device from the CTA's shared-memory image; the host
// emulation reads the transposed entry that slot holds from the transposed table, so it replays which entries the
// kernels keep and the zeta step.  (The image itself is checked against the transposed order by
// tests/test_ntt_resident_image.py.)
HE_HD ulonglong2 ld_tw_image(const RowMod &m, int kp, int tau, int T) {
#if defined(__CUDA_ARCH__)
    return ld_tw_cached(m, T + kp * T + tau);
#else
    return m.tw_t()[(m.scale_mode < 0 ? fwd_image_k(kp) : inv_image_k(kp)) * T + tau];
#endif
}
HE_HD u64 ld_u64(const u64 *p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// ------------------------------------------------------------------------------------------------ arithmetic
// 32-bit limb access.  On the device these are register renames (mov.b64 pack / unpack), which keeps the compiler
// from turning the limb bookkeeping into 64-bit shifts, ORs and carry chains.
HE_HD u64 pack64(u32 lo, u32 hi) {
#if defined(__CUDA_ARCH__)
    u64 v;
    asm("mov.b64 %0, {%1, %2};" : "=l"(v) : "r"(lo), "r"(hi));
    return v;
#else
    return ((u64)hi << 32) | lo;
#endif
}
HE_HD void unpack64(u64 v, u32 &lo, u32 &hi) {
#if defined(__CUDA_ARCH__)
    asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
#else
    lo = (u32)v;
    hi = (u32)(v >> 32);
#endif
}
HE_HD u64 mul_wide_u32(u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    u64 d;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(d) : "r"(a), "r"(b));
    return d;
#else
    return (u64)a * b;
#endif
}
HE_HD u64 mad_wide_u32(u32 a, u32 b, u64 c) {
#if defined(__CUDA_ARCH__)
    u64 d;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
#else
    return (u64)a * b + c;
#endif
}
HE_HD u32 mul_hi_u32(u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (u32)(((u64)a * b) >> 32);
#endif
}

// y w mod p in [0, 4p) for ANY y < 2^64: Shoup with the under-estimated quotient (see the header comment)
//     q~ = y1 w'1 + hi32(y1 w'0) + hi32(y0 w'1),      v = lo64(y w + q~ (2^64 - p)).
// The integer-multiply pipe is the bottleneck (IMAD.WIDE / IMAD.HI occupy it for 4 cycles per warp, IMAD for 2;
// tools/mb_r2.cu measures the butterfly alone), so the sequence is spelled out in PTX: 5 IMAD.WIDE + 4 IMAD and 4-5
// carry adds on the ALU pipe, no register moves.  (The compiler's 64-bit mulhi is 7 wide multiplies plus moves, and
// it re-associates the C version of this into longer, move-heavy code.)
HE_HD u64 shoup4(u64 y, u64 w, u64 wp, u64 np) {
#if defined(__CUDA_ARCH__)
    u64 v;
    asm volatile("{\n\t"
        ".reg .u32 y0, y1, w0, w1, p0, p1, n0, n1, a1, b1, q0, q1, v0, v1, z;\n\t"
        ".reg .u64 A, B, Q, V;\n\t"
        "mov.b64 {y0, y1}, %1;\n\t"
        "mov.b64 {w0, w1}, %2;\n\t"
        "mov.b64 {p0, p1}, %3;\n\t"
        "mov.b64 {n0, n1}, %4;\n\t"
        "mul.hi.u32 a1, y1, p0;\n\t"
        "mul.hi.u32 b1, y0, p1;\n\t"
        "mov.u32 z, 0;\n\t"
        "mov.b64 A, {a1, z};\n\t"
        "mov.b64 B, {b1, z};\n\t"
        "mad.wide.u32 Q, y1, p1, A;\n\t"
        "add.u64 Q, Q, B;\n\t"
        "mov.b64 {q0, q1}, Q;\n\t"
        "mul.wide.u32 V, y0, w0;\n\t"
        "mad.wide.u32 V, q0, n0, V;\n\t"
        "mov.b64 {v0, v1}, V;\n\t"
        "mad.lo.u32 v1, y1, w0, v1;\n\t"
        "mad.lo.u32 v1, y0, w1, v1;\n\t"
        "mad.lo.u32 v1, q1, n0, v1;\n\t"
        "mad.lo.u32 v1, q0, n1, v1;\n\t"
        "mov.b64 %0, {v0, v1};\n\t}"
        : "=l"(v)
        : "l"(y), "l"(w), "l"(wp), "l"(np));
    return v;
#else
    const u32 y0 = (u32)y, y1 = (u32)(y >> 32), wp0 = (u32)wp, wp1 = (u32)(wp >> 32);
    const u64 q = (u64)y1 * wp1 + (((u64)y1 * wp0) >> 32) + (((u64)y0 * wp1) >> 32);
    return y * w + q * np;
#endif
}
// the same for p = h 2^32 + 1: q~ p = q~ + ((q~0 h) << 32) mod 2^64; nh = -h mod 2^32 (= high word of 2^64 - p, plus 1)
HE_HD u64 shoup4h(u64 y, u64 w, u64 wp, u64 np) {
#if defined(__CUDA_ARCH__)
    u64 v;
    asm volatile("{\n\t"
        ".reg .u32 y0, y1, w0, w1, p0, p1, n0, n1, nh, a1, b1, q0, q1, v0, v1, z;\n\t"
        ".reg .u64 A, B, Q, V;\n\t"
        "mov.b64 {y0, y1}, %1;\n\t"
        "mov.b64 {w0, w1}, %2;\n\t"
        "mov.b64 {p0, p1}, %3;\n\t"
        "mov.b64 {n0, n1}, %4;\n\t"
        "add.u32 nh, n1, 1;\n\t"
        "mul.hi.u32 a1, y1, p0;\n\t"
        "mul.hi.u32 b1, y0, p1;\n\t"
        "mov.u32 z, 0;\n\t"
        "mov.b64 A, {a1, z};\n\t"
        "mov.b64 B, {b1, z};\n\t"
        "mad.wide.u32 Q, y1, p1, A;\n\t"
        "add.u64 Q, Q, B;\n\t"
        "mov.b64 {q0, q1}, Q;\n\t"
        "mul.wide.u32 V, y0, w0;\n\t"
        "mov.b64 {v0, v1}, V;\n\t"
        "mad.lo.u32 v1, y1, w0, v1;\n\t"
        "mad.lo.u32 v1, y0, w1, v1;\n\t"
        "mad.lo.u32 v1, q0, nh, v1;\n\t"
        "sub.cc.u32 v0, v0, q0;\n\t"
        "subc.u32 v1, v1, q1;\n\t"
        "mov.b64 %0, {v0, v1};\n\t}"
        : "=l"(v)
        : "l"(y), "l"(w), "l"(wp), "l"(np));
    return v;
#else
    const u32 y0 = (u32)y, y1 = (u32)(y >> 32), wp0 = (u32)wp, wp1 = (u32)(wp >> 32);
    const u64 q = (u64)y1 * wp1 + (((u64)y1 * wp0) >> 32) + (((u64)y0 * wp1) >> 32);
    const u64 h = (0 - np) >> 32;
    return y * w - q - ((u64)((u32)q * (u32)h) << 32);
#endif
}
template <int CLS>
HE_HD u64 shoup4c(u64 y, u64 w, u64 wp, u64 np) { return CLS == kNarrowH ? shoup4h(y, w, wp, np) : shoup4(y, w, wp, np); }
// exact quotient: y w mod p in [0, 2p)
HE_HD u64 shoup2(u64 y, u64 w, u64 wp, u64 np) { return y * w + mulhi64(y, wp) * np; }

// x mod p for x < min(2^64, 512 p): quotient estimated from the top bits with one 32-bit multiply (never above,
// at most 1 below), then one conditional subtraction.
HE_HD u64 reduce_small(u64 x, const u64 p, const u64 np, const int red_shift, const u32 red_recip) {
    const u32 xs = (u32)(x >> red_shift);                   // < 2^21
    const u32 qhat = mul_hi_u32(xs, red_recip);             // floor(x / p) or one less
    u32 np0, np1, rl, rh;
    unpack64(np, np0, np1);
    unpack64(mad_wide_u32(qhat, np0, x), rl, rh);           // x - qhat p  (mod 2^64), in [0, 2p)
    rh = qhat * np1 + rh;
    return csub(pack64(rl, rh), p);
}
HE_HD void reduce_small16(u64 (&x)[16], const RowMod &m) {
    const int shift = m.slot->red_shift;
    const u32 recip = m.slot->red_recip;
    const u64 p = 0 - m.np;
#pragma unroll
    for (int r = 0; r < 16; ++r) x[r] = reduce_small(x[r], p, m.np, shift, recip);
}

// ---- SMALL class: 32-bit Harvey butterflies on zero-extended residues
HE_HD u32 csub32(u32 x, u32 m) {  // x < 2m  ->  x mod m   (unsigned wrap-around makes x - m huge when x < m)
    const u32 d = x - m;
    return d < x ? d : x;
}
HE_HD u32 shoup32(u32 y, u32 w, u32 wp, u32 p) {  // y w mod p in [0, 2p) for any y < 2^32
    return y * w - mul_hi_u32(y, wp) * p;
}

// y w mod p with the class's twiddle product, landing where the butterflies' products land: SMALL [0, 2p) for any
// y < 2^32, NARROW / NARROW-H / MID [0, 4p) and WIDE [0, 2p) for any y < 2^64
template <int CLS>
HE_HD u64 tw_mul(u64 y, const ulonglong2 w, const RowMod &m) {
    if (CLS == kSmall) return shoup32((u32)y, (u32)w.x, (u32)(w.y >> 32), (u32)(0 - m.np));
    if (narrow_like(CLS)) return shoup4c<CLS>(y, w.x, w.y, m.np);
    if (CLS == kMid) return shoup4(y, w.x, w.y, m.np);
    return shoup2(y, w.x, w.y, m.np);
}

template <int CLS>
HE_HD void ct_butterfly(u64 &x, u64 &y, const ulonglong2 w, const RowMod &m) {
    if (CLS == kSmall) {  // [0, 4p) < 2^32
        const u32 p = (u32)(0 - m.np), p2 = 2 * p;
        const u32 xr = csub32((u32)x, p2);
        const u32 v = shoup32((u32)y, (u32)w.x, (u32)(w.y >> 32), p);
        x = xr + v;
        y = xr - v + p2;
    } else if (narrow_like(CLS)) {  // no reduction: x grows by < 4p per stage
        const u64 v = shoup4c<CLS>(y, w.x, w.y, m.np);
        const u64 xo = x + v;
        y = x - v + m.kp;
        x = xo;
    } else if (CLS == kMid) {  // [0, 8p)
        const u64 xr = csub(x, m.kp);
        const u64 v = shoup4(y, w.x, w.y, m.np);
        x = xr + v;
        y = xr - v + m.kp;
    } else {  // [0, 4p), exact quotient
        const u64 xr = csub(x, m.kp);
        const u64 v = shoup2(y, w.x, w.y, m.np);
        x = xr + v;
        y = xr - v + m.kp;
    }
}

// one forward stage (local index J).  The stage index is a template parameter, like the inverse's, so every loop below
// has a compile-time trip count and fully unrolls: with a run-time stage loop around them the register array x got
// an address and lived in local memory.
template <int LOGN, int LB, int C, int CLS, int J>
HE_HD void fwd_stage(u64 (&x)[16], int tau, const RowMod &m) {
    constexpr int E = pass_e(LB, C), F = 1 << E, S0 = LOGN - LB - C, T = (1 << LOGN) / 16;
    constexpr int H = 1 << (C - 1 - J);
    constexpr bool kImage = LB == 0 && resident_twiddles(LOGN);  // LB == 0 twiddles from the resident image
    constexpr bool kZeta = kImage && J == 3;                       // the stage with N/2 twiddles: odd groups via zeta
    const int hi = tau >> (LB - E);
    const ulonglong2 *tw_t = LB == 0 && !kImage ? m.tw_t() + tau : nullptr;
    const ulonglong2 zeta = kZeta ? ld_tw_cached(m, 1) : make_ulonglong2(0, 0);
    ulonglong2 w = make_ulonglong2(0, 0);
#pragma unroll
    for (int grp = 0; grp < (1 << J); ++grp) {
        const bool odd = kZeta && (grp & 1);  // w_grp = w_(grp-1) zeta: keep the even group's twiddle
        if (!odd)
            w = kImage  ? ld_tw_image(m, kZeta ? 7 + grp / 2 : (1 << J) - 1 + grp, tau, T)
                : LB == 0 ? ld_tw(tw_t + ((1 << J) - 1 + grp) * T)
                          : ld_tw_cached(m, (1 << (S0 + J)) + (hi << J) + grp);
#pragma unroll
        for (int k = 0; k < H; ++k) {
            const int a = grp * 2 * H + k;
#pragma unroll
            for (int f = 0; f < F; ++f) {
                if (odd) x[(a + H) * F + f] = tw_mul<CLS>(x[(a + H) * F + f], zeta, m);
                ct_butterfly<CLS>(x[a * F + f], x[(a + H) * F + f], w, m);
            }
        }
    }
}
template <int LOGN, int LB, int C, int CLS>
HE_HD void fwd_pass(u64 (&x)[16], int tau, const RowMod &m) {
    fwd_stage<LOGN, LB, C, CLS, 0>(x, tau, m);
    if (C > 1) fwd_stage<LOGN, LB, C, CLS, (C > 1 ? 1 : 0)>(x, tau, m);
    if (C > 2) fwd_stage<LOGN, LB, C, CLS, (C > 2 ? 2 : 0)>(x, tau, m);
    if (C > 3) fwd_stage<LOGN, LB, C, CLS, (C > 3 ? 3 : 0)>(x, tau, m);
}

// reduce the outputs of the last forward stage to canonical residues
template <int CLS>
HE_HD void fwd_finish(u64 (&x)[16], const RowMod &m) {
    if (CLS == kSmall) {
        const u32 p = (u32)(0 - m.np);
#pragma unroll
        for (int r = 0; r < 16; ++r) x[r] = csub32(csub32((u32)x[r], 2 * p), p);
    } else {
        reduce_small16(x, m);  // NARROW < (2 + 4 LOGN) p, MID < 8p, WIDE < 4p
    }
}

// ------------------------------------------------------------------------------------------------ inverse
// zeta (non-null): the difference is multiplied by *zeta before w (an odd group of the resident image's zeta stage)
template <int CLS>
HE_HD void gs_butterfly(u64 &x, u64 &y, const ulonglong2 w, const RowMod &m, u64 kp, const ulonglong2 *zeta = nullptr) {
    if (CLS == kSmall) {  // inputs < 2p, outputs < 2p
        const u32 p = (u32)(0 - m.np), p2 = 2 * p;
        const u32 s = csub32((u32)x + (u32)y, p2);
        u32 d = (u32)x - (u32)y + p2;
        if (zeta) d = (u32)tw_mul<CLS>(d, *zeta, m);
        y = shoup32(d, (u32)w.x, (u32)(w.y >> 32), p);
        x = s;
    } else if (narrow_like(CLS)) {  // inputs < kp (a multiple of p), outputs x < 2 kp, y < 4p
        const u64 s = x + y;
        u64 d = x - y + kp;
        if (zeta) d = tw_mul<CLS>(d, *zeta, m);
        y = shoup4c<CLS>(d, w.x, w.y, m.np);
        x = s;
    } else if (CLS == kMid) {  // inputs < 4p, outputs < 4p
        const u64 s = csub(x + y, kp);
        u64 d = x - y + kp;
        if (zeta) d = tw_mul<CLS>(d, *zeta, m);
        y = shoup4(d, w.x, w.y, m.np);
        x = s;
    } else {  // inputs < 2p, outputs < 2p
        const u64 s = csub(x + y, kp);
        u64 d = x - y + kp;
        if (zeta) d = tw_mul<CLS>(d, *zeta, m);
        y = shoup2(d, w.x, w.y, m.np);
        x = s;
    }
}

// one inverse stage (local index J)
template <int LOGN, int LB, int C, int CLS, int BIN, int J>
HE_HD void inv_stage(u64 (&x)[16], const int tau, const RowMod &m) {
    constexpr int E = pass_e(LB, C), F = 1 << E, T = (1 << LOGN) / 16;
    constexpr int HH = 1 << J;
    constexpr bool kLast = (LB + J == LOGN - 1);
    constexpr int kGroups = 1 << (LOGN - 1 - LB - J);
    const int hi = tau >> (LB - E);
    const u64 kp = narrow_like(CLS) ? (0 - m.np) * (u64)inv_bound_after(BIN, J) : m.kp;  // inputs < kp
    constexpr bool kImage = LB == 0 && resident_twiddles(LOGN);  // LB == 0 twiddles from the resident image
    constexpr bool kZeta = kImage && J == 0;                       // the stage with N/2 twiddles: odd groups via zeta
    const ulonglong2 *tw_t = LB == 0 && !kImage ? m.tw_t() + tau : nullptr;
    const ulonglong2 zeta = kZeta ? ld_tw_cached(m, 1) : make_ulonglong2(0, 0);
    ulonglong2 w = make_ulonglong2(0, 0);
#pragma unroll
    for (int grp = 0; grp < (1 << (C - 1 - J)); ++grp) {
        if (!kLast || m.partial) {
            const bool odd = kZeta && (grp & 1);  // w_grp = w_(grp-1) zeta: keep the even group's twiddle
            // LB == 0: entry index inside the thread's 15 = (groups of the earlier stages) + grp
            if (!odd)
                w = kImage  ? ld_tw_image(m, kZeta ? grp / 2 : 16 - (16 >> J) + grp - 4, tau, T)
                    : LB == 0 ? ld_tw(tw_t + (16 - (16 >> J) + grp) * T)
                              : ld_tw_cached(m, kGroups + (hi << (C - 1 - J)) + grp);
#pragma unroll
            for (int k = 0; k < HH; ++k) {
                const int a = grp * 2 * HH + k;
#pragma unroll
                for (int f = 0; f < F; ++f) gs_butterfly<CLS>(x[a * F + f], x[(a + HH) * F + f], w, m, kp, odd ? &zeta : nullptr);
            }
        } else {
            const u64 *sc = &m.slot->inv_scale[m.scale_mode].c0;  // c0, c0p, c1, c1p
            const u64 c0 = ld_u64(sc), c0p = ld_u64(sc + 1), c1 = ld_u64(sc + 2), c1p = ld_u64(sc + 3);
#pragma unroll
            for (int k = 0; k < HH; ++k) {
                const int a = grp * 2 * HH + k;
#pragma unroll
                for (int f = 0; f < F; ++f) {
                    if (CLS == kSmall) {
                        const u32 p = (u32)(0 - m.np);
                        const u32 xa = (u32)x[a * F + f], ya = (u32)x[(a + HH) * F + f];
                        x[a * F + f] = csub32(shoup32(xa + ya, (u32)c0, (u32)(c0p >> 32), p), p);
                        x[(a + HH) * F + f] = csub32(shoup32(xa - ya + 2 * p, (u32)c1, (u32)(c1p >> 32), p), p);
                        continue;
                    }
                    const u64 xa = x[a * F + f], ya = x[(a + HH) * F + f];
                    const u64 s = xa + ya;          // NARROW < 2 kp <= 2^64, MID < 8p, WIDE < 4p
                    const u64 d = xa - ya + kp;
                    x[a * F + f] = csub(shoup2(s, c0, c0p, m.np), 0 - m.np);         // (x + y) N^-1     (PolyRq+Ntt.swift:416-419)
                    x[(a + HH) * F + f] = csub(shoup2(d, c1, c1p, m.np), 0 - m.np);  // (x - y) N^-1 psi^-(N/2)
                }
            }
        }
    }
}

// BIN = bound (units of p) on the pass inputs (NARROW only; ignored otherwise)
template <int LOGN, int LB, int C, int CLS, int BIN>
HE_HD void inv_pass(u64 (&x)[16], int tau, const RowMod &m) {
    inv_stage<LOGN, LB, C, CLS, BIN, 0>(x, tau, m);
    if (C > 1) inv_stage<LOGN, LB, C, CLS, BIN, (C > 1 ? 1 : 0)>(x, tau, m);
    if (C > 2) inv_stage<LOGN, LB, C, CLS, BIN, (C > 2 ? 2 : 0)>(x, tau, m);
    if (C > 3) inv_stage<LOGN, LB, C, CLS, BIN, (C > 3 ? 3 : 0)>(x, tau, m);
}

HE_HD void inv_reduce(u64 (&x)[16], const RowMod &m) { reduce_small16(x, m); }  // < 512 p

// ---- transposed twiddle tables for the LB == 0 pass (built on the host by context.cu, checked by the emulation)
// forward: thread tau, stage j (0..3), group grp (< 2^j): entry (2^j - 1 + grp) = tw[2^(LOGN-4+j) + (tau << j) + grp]
HE_HD int fwd_last_source(int logn, int k, int tau) {
    int j = 0;
    while ((2 << j) - 1 <= k) ++j;
    const int grp = k - ((1 << j) - 1);
    return (1 << (logn - 4 + j)) + (tau << j) + grp;
}
// inverse: stage J (0..3), group grp (< 2^(3-J)): entry (16 - (16 >> J) + grp) = itw[2^(LOGN-1-J) + (tau << (3-J)) + grp]
HE_HD int inv_first_source(int logn, int k, int tau) {
    int J = 0;
    while (16 - (16 >> (J + 1)) <= k) ++J;
    const int grp = k - (16 - (16 >> J));
    return (1 << (logn - 1 - J)) + (tau << (3 - J)) + grp;
}
// the resident image (resident_twiddles): entry i (< image_entries) = tw[image_source(logn, false, i)] forward,
// itw[image_source(logn, true, i)] inverse
HE_HD int image_source(int logn, bool inverse, int i) {
    const int T = 1 << (logn - 4);
    if (i < T) return i;
    const int kp = i / T - 1, tau = i % T;
    return inverse ? inv_first_source(logn, inv_image_k(kp), tau) : fwd_last_source(logn, fwd_image_k(kp), tau);
}

}  // namespace fast
}  // namespace hecuda
