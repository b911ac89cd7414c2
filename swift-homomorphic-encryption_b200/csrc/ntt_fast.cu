// ntt_fast.cu -- sm_90a kernels of the register-tiled NTT (see ntt_fast.cuh for the pass structure).
//
// Persistent CTAs: each CTA (T = N/16 threads; as many CTAs per SM as the register budget of ntt_min_ctas allows) walks
// over rows task = blockIdx.x, blockIdx.x + gridDim.x, ...  For every row
//   1. TMA in: one thread issues bulk-tensor copies (cp.async.bulk.tensor.2d, 256 lines = 32 KB each, 128-byte
//      swizzle) that land a row in a shared-memory row buffer and complete on that buffer's mbarrier -- with two
//      buffers (N = 2^13, ntt_row_buffers) the CTA's next row, otherwise this row; it also prefetches the row after
//      that into L2 (cp.async.bulk.prefetch.tensor) and, when the row's modulus differs from the previous row's,
//      bulk-copies the first N/16 twiddles (all the LB > 0 passes need; at N = 2^13 the resident image of all the
//      twiddles, ntt_fast.cuh) into the CTA's shared-memory twiddle cache;
//   2. 3-4 register passes over the row in shared memory (ntt_fast.cuh), one __syncthreads between passes;
//   3. TMA out: bulk-tensor copies shared -> global of the finished row (same swizzle, undone by the copy engine), one
//      bulk group per row; a buffer is refilled once the copy engine has read it.
// NARROW / MID / WIDE rows (different lazy-reduction schedules) are mixed in one launch: the row's class selects the
// instruction stream, rows are ordered class-major so all CTAs walk the classes in step, and there is one tail per
// NTT call instead of one per class.  Each kernel is compiled for a class set (ntt_fast.cuh): the all-class set, and at
// N = 2^13 also NARROW + NARROW-H for the multiply's rows.
#include <cuda.h>

#include <mutex>

#include <algorithm>
#include "kernels.cuh"
#include "ntt_fast.cuh"

namespace hecuda {
using namespace fast;

constexpr int kMaxRowList = 2 * (kMaxL + 1) * kMaxL;  // key-switch digit rows: (l + 1) * l, twice that as half rows of N = 2^15
struct RowList {          // rows (within a polynomial) that one launch handles
    int rows_per_poly;
    int count;
    unsigned short row[kMaxRowList];
    unsigned short slot[kMaxRowList];  // (virtual slots of N = 2^15 exceed a byte at 32 moduli)
    // 3 bits class | bit 3: re-reduce the gathered input into this row's modulus (forward only) | bit 4: half of a
    // 2^15 row (inverse only: no N^-1 scaling)
    unsigned char flags[kMaxRowList];
    unsigned short src_row[kMaxRowList];  // input side (forward only): source row
    long long src_poly_stride;           // words between consecutive input polynomials
};

// ------------------------------------------------------------------------------------------------ TMA / mbarrier
__device__ __forceinline__ u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(u64 *bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity) {
    asm volatile(
        "{\n\t.reg .pred done;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n\t"
        "@!done bra WAIT_%=;\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D bulk copy global -> shared (twiddle cache), completes `bytes` on the mbarrier
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, u32 bytes, u64 *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// one box (16 words x kBoxLines lines) of the 2-D view {word in line, line} of a buffer, global -> shared
__device__ __forceinline__ void tma_load_box(void *smem_dst, const CUtensorMap *map, int line, u64 *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(0), "r"(line), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_store_box(const CUtensorMap *map, int line, const void *smem_src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(map), "r"(0), "r"(line),
                 "r"(smem_u32(smem_src))
                 : "memory");
}
__device__ __forceinline__ void tma_prefetch_box(const CUtensorMap *map, int line) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(map), "r"(0), "r"(line) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the copy engine has read the buffers of all but the PENDING most recently committed store groups
template <int PENDING>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(PENDING) : "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ row bodies
template <int LOGN, int CLS, int K>
__device__ __forceinline__ void fwd_row_pass(u64 (&x)[16], u64 *sm, int tau, const RowMod &m, bool reduce_in) {
    constexpr int P = plan_passes(LOGN), C = fwd_c(LOGN, K), LB = fwd_lb(LOGN, K);
    load_smem<LOGN, LB, C>(x, sm, tau);
    if (K == 0 && reduce_in) {  // gathered key-switch digit whose source modulus is too large for the lazy range
#pragma unroll
        for (int r = 0; r < 16; ++r) x[r] = barrett64(x[r], 0 - m.np, m.slot->mu1);
    }
    fwd_pass<LOGN, LB, C, CLS>(x, tau, m);
    if (K == P - 1) fwd_finish<CLS>(x, m);
    store_smem<LOGN, LB, C>(x, sm, tau);
}
template <int LOGN, int CLS>
__device__ __forceinline__ void fwd_row(u64 *sm, int tau, const RowMod &m, bool reduce_in) {
    constexpr int P = plan_passes(LOGN);
    u64 x[16];
    fwd_row_pass<LOGN, CLS, 0>(x, sm, tau, m, reduce_in);
    __syncthreads();
    fwd_row_pass<LOGN, CLS, 1>(x, sm, tau, m, false);
    __syncthreads();
    if (P == 4) {
        fwd_row_pass<LOGN, CLS, (P == 4 ? 2 : 1)>(x, sm, tau, m, false);
        __syncthreads();
    }
    fwd_row_pass<LOGN, CLS, P - 1>(x, sm, tau, m, false);
}

template <int LOGN, int CLS, int K>
__device__ __forceinline__ void inv_row_pass(u64 (&x)[16], u64 *sm, int tau, const RowMod &m) {
    constexpr int C = inv_c(LOGN, K), LB = inv_lb(LOGN, K);
    load_smem<LOGN, LB, C>(x, sm, tau);
    if (narrow_like(CLS) && K > 0 && inv_reduce_at(LOGN, K)) inv_reduce(x, m);
    inv_pass<LOGN, LB, C, CLS, inv_bound_in(LOGN, K)>(x, tau, m);
    if (K == plan_passes(LOGN) - 1 && m.partial) {  // half of a 2^15 row: hand canonical residues to the merge kernel
        if (CLS == kSmall) {
#pragma unroll
            for (int r = 0; r < 16; ++r) x[r] = csub32((u32)x[r], (u32)(0 - m.np));
        } else {
            reduce_small16(x, m);  // NARROW < 512 p, MID < 4p, WIDE < 2p
        }
    }
    store_smem<LOGN, LB, C>(x, sm, tau);
}
template <int LOGN, int CLS>
__device__ __forceinline__ void inv_row(u64 *sm, int tau, const RowMod &m) {
    constexpr int P = plan_passes(LOGN);
    u64 x[16];
    inv_row_pass<LOGN, CLS, 0>(x, sm, tau, m);
    __syncthreads();
    inv_row_pass<LOGN, CLS, 1>(x, sm, tau, m);
    __syncthreads();
    if (P == 4) {
        inv_row_pass<LOGN, CLS, (P == 4 ? 2 : 1)>(x, sm, tau, m);
        __syncthreads();
    }
    inv_row_pass<LOGN, CLS, P - 1>(x, sm, tau, m);
}

// the instruction stream of a row of class `cls` among the streams of the class set CLASSES (ntt_fast.cuh); a row whose
// class is not in the set is a launcher error, except NARROW-H, which takes NARROW's stream when the set lacks its own
template <int LOGN, unsigned CLASSES>
__device__ __forceinline__ void fwd_row_of(int cls, u64 *sm, int tau, const RowMod &m, bool reduce_in) {
    if (has_class(CLASSES, kNarrowH) && cls == kNarrowH) fwd_row<LOGN, kNarrowH>(sm, tau, m, reduce_in);
    else if (has_class(CLASSES, kNarrow) && narrow_like(cls)) fwd_row<LOGN, kNarrow>(sm, tau, m, reduce_in);
    else if (has_class(CLASSES, kSmall) && cls == kSmall) fwd_row<LOGN, kSmall>(sm, tau, m, reduce_in);
    else if (has_class(CLASSES, kMid) && cls == kMid) fwd_row<LOGN, kMid>(sm, tau, m, reduce_in);
    else if (has_class(CLASSES, kWide)) fwd_row<LOGN, kWide>(sm, tau, m, reduce_in);
}
template <int LOGN, unsigned CLASSES>
__device__ __forceinline__ void inv_row_of(int cls, u64 *sm, int tau, const RowMod &m) {
    if (has_class(CLASSES, kNarrowH) && cls == kNarrowH) inv_row<LOGN, kNarrowH>(sm, tau, m);
    else if (has_class(CLASSES, kNarrow) && narrow_like(cls)) inv_row<LOGN, kNarrow>(sm, tau, m);
    else if (has_class(CLASSES, kSmall) && cls == kSmall) inv_row<LOGN, kSmall>(sm, tau, m);
    else if (has_class(CLASSES, kMid) && cls == kMid) inv_row<LOGN, kMid>(sm, tau, m);
    else if (has_class(CLASSES, kWide)) inv_row<LOGN, kWide>(sm, tau, m);
}

// Row buffers of a CTA.  With one CTA per SM (N = 2^13) nothing else on the SM runs while the CTA waits for its copies,
// so the next row's TMA-in and the previous row's TMA-out run under the current row's butterflies (C2 on H100 at a
// 400 W power limit: +4 % over one buffer; three buffers measured 1-2 % behind two).  With several CTAs per SM
// (N <= 2^12) the other CTAs fill those gaps, and at N = 2^14 a second 128 KB buffer does not fit.
HE_HD constexpr int ntt_row_buffers(int logn) { return logn == 13 ? 2 : 1; }
// The twiddle cache of a CTA: at N = 2^13 (resident_twiddles, ntt_fast.cuh) the resident image of every twiddle the
// transform reads (96 KB: the two row buffers leave just room for it), otherwise the first N/16 twiddles (the LB > 0
// passes; the LB == 0 pass reads the transposed table in global memory).  Both arrive by one 1-D bulk copy.
template <int LOGN>
HE_HD constexpr u32 ntt_twiddle_bytes() {
    return (u32)sizeof(ulonglong2) * (resident_twiddles(LOGN) ? image_entries(LOGN) : 1 << (LOGN - 4));
}
// cp.async.bulk moves a multiple of 16 bytes, and an mbarrier's pending transaction count stays below 2^20
static_assert(ntt_twiddle_bytes<13>() == 98304 && ntt_twiddle_bytes<13>() % 16 == 0 && ntt_twiddle_bytes<13>() < (1u << 20),
              "the resident image is one 1-D bulk copy on one mbarrier");
template <int LOGN, bool INVERSE>
__device__ __forceinline__ const ulonglong2 *ntt_twiddle_source(const ModSlot &S) {
    if (resident_twiddles(LOGN)) return INVERSE ? S.itw_img : S.tw_img;
    return INVERSE ? S.itw : S.tw;
}

// Shared memory of a CTA: [row buffers: B x N words][twiddle cache][B + 1 mbarriers].
template <int LOGN>
constexpr size_t ntt_smem_bytes() {
    constexpr int B = ntt_row_buffers(LOGN);
    return sizeof(u64) * B * ((size_t)1 << LOGN) + ntt_twiddle_bytes<LOGN>() + sizeof(u64) * (B + 1);
}
static_assert(ntt_smem_bytes<13>() == 229400 && ntt_smem_bytes<13>() <= 232448, "N = 2^13: 227 KB of shared memory a CTA");

// CTAs per SM the register budget is sized for.  1024 threads per SM (64 registers a thread, some spills) except at
// N = 2^13, where one 512-thread CTA with 128 registers and no spills is faster on H100 (C2, runs alternated in one
// session: +2.7 % at a 700 W power limit, +6 % at 400 W; DESIGN.md section 4); at 64 registers that kernel still spills
// (about 450 bytes a thread), and its two row buffers (136 KB) leave room for one CTA per SM in any case.  At N = 2^12
// the 64-register budget beat 80 and 128 registers by 3-4 % (C1, C2-u32).
constexpr int ntt_min_ctas(int logn) { return logn == 13 ? 1 : 1024 / ((1 << logn) / 16); }

template <int LOGN, bool INVERSE, unsigned CLASSES>
__global__ void __launch_bounds__((1 << LOGN) / 16, ntt_min_ctas(LOGN))
    ntt_rows_kernel(const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_out,
                    const ModSlot *__restrict__ slots, const __grid_constant__ RowList rl, const int polys,
                    const int scale_mode) {
    extern __shared__ __align__(1024) u64 smem[];  // row buffers first: the 128-byte swizzle wants them 1024-byte aligned
    constexpr int kLines = (1 << LOGN) / kLineWords;
    constexpr int kBoxes = kLines > kBoxLines ? kLines / kBoxLines : 1;
    constexpr int kLinesPerBox = kLines / kBoxes;
    constexpr u32 kRowBytes = (u32)sizeof(u64) << LOGN, kTwBytes = ntt_twiddle_bytes<LOGN>();
    // B row buffers; row k of the CTA uses buffer k % B, and its TMA-in is issued AHEAD rows before the CTA starts on it
    constexpr int B = ntt_row_buffers(LOGN), AHEAD = B > 1 ? 1 : 0;
    ulonglong2 *tw_cache = reinterpret_cast<ulonglong2 *>(smem + B * (1 << LOGN));
    u64 *bar_row = reinterpret_cast<u64 *>(tw_cache + kTwBytes / sizeof(ulonglong2));  // one per buffer
    u64 *bar_tw = bar_row + B;
    const int tau = threadIdx.x;
    const int tasks = polys * rl.count;  // < 2^31 (checked by the launcher)
    // global position (in 16-word lines) of task t's input row
    auto in_line = [&](int t) {
        const int w = t / polys, p = t - w * polys;
        const int64_t word = INVERSE ? ((int64_t)p * rl.rows_per_poly + rl.row[w]) << LOGN
                                     : (int64_t)p * rl.src_poly_stride + ((int64_t)rl.src_row[w] << LOGN);
        return (int)(word >> 4);
    };
    auto load_row = [&](int t, int buf) {
        mbar_arrive_expect_tx(&bar_row[buf], kRowBytes);
        const int line = in_line(t);
        u64 *dst = smem + buf * (1 << LOGN);
#pragma unroll
        for (int b = 0; b < kBoxes; ++b) tma_load_box(dst + b * kLinesPerBox * kLineWords, &map_in, line + b * kLinesPerBox, &bar_row[buf]);
    };
    if (tau == 0) {
        if (smem_u32(smem) & 1023) __trap();  // dynamic shared memory starts at the window base when there is no static part
#pragma unroll
        for (int b = 0; b < B; ++b) mbar_init(&bar_row[b], 1);
        mbar_init(bar_tw, 1);
        if (AHEAD && (int)blockIdx.x < tasks) load_row(blockIdx.x, 0);
    }
    __syncthreads();
    u32 phase_row = 0, phase_tw = 0;  // phase_row: bit b = parity of buffer b's next completion
    int cached_slot = -1;
    int buf = 0;
    for (int task = blockIdx.x; task < tasks; task += gridDim.x) {
        const int which = task / polys;
        const int poly = task - which * polys;
        const int flags = rl.flags[which];
        const int slot = rl.slot[which];
        const ModSlot &S = slots[slot];
        u64 *sm = smem + buf * (1 << LOGN);
        // line index (16-word lines) of the row inside the buffer each tensor map describes
        const int64_t out_word = ((int64_t)poly * rl.rows_per_poly + rl.row[which]) << LOGN;
        const bool new_slot = slot != cached_slot;  // uniform over the CTA
        cached_slot = slot;
        if (tau == 0) {
            // every thread has passed the barrier that follows its last use of the twiddle cache
            if (new_slot) {
                mbar_arrive_expect_tx(bar_tw, kTwBytes);
                tma_load_1d(tw_cache, ntt_twiddle_source<LOGN, INVERSE>(S), kTwBytes, bar_tw);
            }
            // the row AHEAD tasks on goes into a buffer whose last row's TMA-out was committed B - AHEAD rows ago: the
            // copy engine must have read it, which leaves the B - 1 - AHEAD stores committed since then in flight
            const int fill = task + AHEAD * gridDim.x;
            if (fill < tasks) {
                tma_store_wait_read<B - 1 - AHEAD>();
                load_row(fill, (buf + AHEAD) % B);
            }
            const int next = fill + gridDim.x;
            if (next < tasks) {  // L2 prefetch of the row after that
                const int line = in_line(next);
#pragma unroll
                for (int b = 0; b < kBoxes; ++b) tma_prefetch_box(&map_in, line + b * kLinesPerBox);
            }
        }
        const int cls = flags & 7;
        RowMod m;
        m.np = 0 - S.p;
        m.kp = (cls == kWide || cls == kSmall) ? 2 * S.p : 4 * S.p;  // (NARROW / NARROW-H / MID: 4p)
        m.tw = nullptr;
        m.tw_s = smem_u32(tw_cache);
        m.slot = &S;
        m.scale_mode = INVERSE ? scale_mode : -1;
        m.partial = INVERSE && (flags & 16) != 0;
        if (new_slot) {
            mbar_wait(bar_tw, phase_tw);
            phase_tw ^= 1;
        }
        mbar_wait(&bar_row[buf], (phase_row >> buf) & 1);
        phase_row ^= 1u << buf;
        if (INVERSE) inv_row_of<LOGN, CLASSES>(cls, sm, tau, m);
        else fwd_row_of<LOGN, CLASSES>(cls, sm, tau, m, (flags & 8) != 0);
        // ---- TMA out: every thread makes its generic-proxy writes visible to the async proxy, then one thread copies
        fence_proxy_async_smem();
        __syncthreads();
        if (tau == 0) {
            const int line = (int)(out_word >> 4);
#pragma unroll
            for (int b = 0; b < kBoxes; ++b) tma_store_box(&map_out, line + b * kLinesPerBox, sm + b * kLinesPerBox * kLineWords);
            tma_commit();  // one group per row: the buffer is refilled once the copy engine has read it (above)
        }
        buf = buf + 1 == B ? 0 : buf + 1;
    }
    if (tau == 0) tma_store_wait_all();
}

// ------------------------------------------------------------------------------------ forward NTT + tensor product
__device__ __forceinline__ u32 cluster_ctarank() {
    u32 r;
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ int cluster_id_x() {
    u32 r;
    asm("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return (int)r;
}
__device__ __forceinline__ int cluster_count_x() {
    u32 r;
    asm("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
    return (int)r;
}
// every thread of the cluster: arrive (release: this thread's shared-memory writes) / wait (acquire)
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// arrive without ordering memory: for a thread whose reads of the peer's rows have all returned (their values are
// used before it arrives); a release here would also wait for this thread's global stores
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
// the address of the same shared-memory location in CTA `rank` of the cluster
__device__ __forceinline__ u32 cluster_map(u32 addr, u32 rank) {
    u32 r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ ulonglong2 ld_cluster_v2(u32 addr) {
    ulonglong2 v;
    asm volatile("ld.shared::cluster.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "r"(addr) : "memory");
    return v;
}
// a b 2^-64 mod p, canonical (behz.cu:tensor_kernel's arithmetic: the inverse NTT's kScaleTMont restores the 2^64);
// H: p = h 2^32 + 1 (mont_reduce_h, the same value)
template <bool H>
__device__ __forceinline__ u64 mont_product(u64 a, u64 b, u64 p, u64 ninv) { return csub(mont_reduce_c<H>((u128)a * b, p, ninv), p); }

// The N = 2^13 ct x ct multiply's forward NTT and tensor product (Bfv+Multiply.swift:51-57, :80-82) in one kernel, so
// the 4 R transformed operand rows of a pair never go to HBM.  A task is one (pair, row r of [Q, aux]); tasks are
// r-major like the row NTT's, so consecutive tasks share the twiddle cache.  Clusters of two CTAs walk the tasks
// persistently, both CTAs the same sequence.  CTA rank k transforms a_k and b_k (polynomial k of lhs and of rhs) into
// its own row buffers, the same TMA-in and register passes as ntt_rows_kernel; then rank 0 computes c0 = a0 b0 and
// rank 1 c2 = a1 b1 from their own rows, and each computes half the columns of c1 = a0 b1 + a1 b0 with the peer's two
// rows read through distributed shared memory.  (Splitting the rows a0 a1 | b0 b1 instead would put a remote operand
// in every product; this split reads N remote words per CTA and task.)  Both CTAs' buffers carry the same 128-byte
// swizzle, so one shared-memory offset holds the same coefficient in all four rows; the products are stored straight
// to `ten` with the swizzle undone, in the layout the inverse NTT reads.
//
// The Q rows (r < L) are read from lhs / rhs themselves, the auxiliary rows from what the lift wrote,
// ext[pair][4][L + 1][N] (polynomials a0 a1 b0 b1).
//
// Shared memory: [row buffers: operand j of the task in buffer j, 2 x N words][twiddle cache: the resident image][3 mbarriers].
// A task's rows stay in their buffers until the cluster barrier that ends its tensor step; the next task's two rows
// are loaded after it, the second under the first one's passes.  (A third buffer that took the next task's first row
// under the current task's second row and tensor step measured no faster: C2 on H100 at a 400 W power limit, three
// runs each, 136.3-137.1 k mult/s with three buffers, 136.3-137.7 k with two.)
template <int LOGN>
constexpr size_t ntt_tensor_smem_bytes() {
    return sizeof(u64) * 2 * ((size_t)1 << LOGN) + ntt_twiddle_bytes<LOGN>() + sizeof(u64) * 3;
}
static_assert(ntt_tensor_smem_bytes<13>() == 229400, "N = 2^13: 227 KB of shared memory a CTA");

// The tensor step of one task: c0 (rank 0) or c2 (rank 1) from this CTA's rows x = a_rank, y = b_rank, then, once the
// peer's rows are final, this CTA's half of the columns of c1.  H: the row's prime is h 2^32 + 1.
template <int LOGN, bool H>
__device__ __forceinline__ void tensor_step(const u64 *x, const u64 *y, u64 *out, int64_t comp, u32 rank, int tau, u64 p, u64 ninv) {
    constexpr int N = 1 << LOGN, T = N / 16;
    u64 *own = out + (rank ? 2 * comp : 0);  // c0 (rank 0) or c2 (rank 1): this CTA's rows only
#pragma unroll 4
    for (int w = 2 * tau; w < N; w += 2 * T) {
        const ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(x + w), b = *reinterpret_cast<const ulonglong2 *>(y + w);
        *reinterpret_cast<ulonglong2 *>(own + smem_phys(w)) =
            make_ulonglong2(mont_product<H>(a.x, b.x, p, ninv), mont_product<H>(a.y, b.y, p, ninv));
    }
    cluster_wait();  // the peer's rows are final
    // c1 = a0 b1 + a1 b0 = x Y + X y over this CTA's half of the columns (X, Y: the peer's rows), summed at 128 bits
    // before its one reduction
    const u32 px = cluster_map(smem_u32(x), rank ^ 1), py = cluster_map(smem_u32(y), rank ^ 1);
#pragma unroll 4
    for (int w = (int)rank * (N / 2) + 2 * tau; w < ((int)rank + 1) * (N / 2); w += 2 * T) {
        const ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(x + w), b = *reinterpret_cast<const ulonglong2 *>(y + w);
        const ulonglong2 A = ld_cluster_v2(px + 8u * w), Bv = ld_cluster_v2(py + 8u * w);
        u128 m0 = (u128)a.x * Bv.x, m1 = (u128)a.y * Bv.y;
        mac128(m0, A.x, b.x);
        mac128(m1, A.y, b.y);
        *reinterpret_cast<ulonglong2 *>(out + comp + smem_phys(w)) =
            make_ulonglong2(csub(mont_reduce_c<H>(m0, p, ninv), p), csub(mont_reduce_c<H>(m1, p, ninv), p));
    }
}

template <int LOGN, unsigned CLASSES>
__global__ void __launch_bounds__((1 << LOGN) / 16, 1)
    ntt_forward_tensor_kernel(const __grid_constant__ CUtensorMap map_lhs, const __grid_constant__ CUtensorMap map_rhs,
                              const __grid_constant__ CUtensorMap map_ext, u64 *__restrict__ ten,
                              const ModSlot *__restrict__ slots, const __grid_constant__ RowList rl, const int items,
                              const int L) {
    extern __shared__ __align__(1024) u64 smem[];  // row buffers first: the 128-byte swizzle wants them 1024-byte aligned
    constexpr int N = 1 << LOGN;
    constexpr int kBoxes = N / kLineWords / kBoxLines;
    constexpr u32 kRowBytes = (u32)sizeof(u64) << LOGN, kTwBytes = ntt_twiddle_bytes<LOGN>();
    static_assert(kBoxes >= 1, "one row is at least one box");
    ulonglong2 *tw_cache = reinterpret_cast<ulonglong2 *>(smem + 2 * N);
    u64 *bar_row = reinterpret_cast<u64 *>(tw_cache + kTwBytes / sizeof(ulonglong2));  // one per buffer
    u64 *bar_tw = bar_row + 2;
    const int tau = threadIdx.x;
    const u32 rank = cluster_ctarank();
    const int first = cluster_id_x(), stride = cluster_count_x();
    const int R = rl.rows_per_poly;
    const int tasks = items * rl.count;  // < 2^31 (checked by the launcher)
    // operand j's row of task t into buffer j: polynomial `rank` of lhs (j = 0) or rhs (j = 1)
    auto load_row = [&](int t, int j) {
        const int w = t / items, item = t - w * items, r = rl.row[w];
        const CUtensorMap *map;
        int64_t word;
        if (r < L) {
            map = j ? &map_rhs : &map_lhs;
            word = ((int64_t)(2 * item + (int)rank) * L + r) << LOGN;
        } else {
            map = &map_ext;
            word = ((int64_t)(4 * item + 2 * j + (int)rank) * (L + 1) + r - L) << LOGN;
        }
        const int line = (int)(word >> 4);
        mbar_arrive_expect_tx(&bar_row[j], kRowBytes);
#pragma unroll
        for (int b = 0; b < kBoxes; ++b) tma_load_box(smem + j * N + b * kBoxLines * kLineWords, map, line + b * kBoxLines, &bar_row[j]);
    };
    if (tau == 0) {
        if (smem_u32(smem) & 1023) __trap();  // dynamic shared memory starts at the window base when there is no static part
        mbar_init(&bar_row[0], 1);
        mbar_init(&bar_row[1], 1);
        mbar_init(bar_tw, 1);
    }
    // both CTAs have started (and initialised their barriers) before either reads the other's shared memory
    cluster_arrive();
    cluster_wait();
    u32 phase_row = 0, phase_tw = 0;  // both row buffers complete once per task
    int cached_slot = -1;
    for (int task = first; task < tasks; task += stride) {
        // the previous task's tensor step is over in both CTAs: its two buffers may be refilled
        if (task != first) cluster_wait();
        const int which = task / items;
        const int item = task - which * items;
        const int slot = rl.slot[which], r = rl.row[which], cls = rl.flags[which] & 7;
        const ModSlot &S = slots[slot];
        const bool new_slot = slot != cached_slot;  // uniform over the cluster
        cached_slot = slot;
        if (tau == 0) {
            // every thread has passed the barrier that follows its last use of the twiddle cache
            if (new_slot) {
                mbar_arrive_expect_tx(bar_tw, kTwBytes);
                tma_load_1d(tw_cache, ntt_twiddle_source<LOGN, false>(S), kTwBytes, bar_tw);
            }
            load_row(task, 0);
            load_row(task, 1);
        }
        RowMod m;
        m.np = 0 - S.p;
        m.kp = (cls == kWide || cls == kSmall) ? 2 * S.p : 4 * S.p;
        m.tw = nullptr;
        m.tw_s = smem_u32(tw_cache);
        m.slot = &S;
        m.scale_mode = -1;
        m.partial = false;
        if (new_slot) {
            mbar_wait(bar_tw, phase_tw);
            phase_tw ^= 1;
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            mbar_wait(&bar_row[j], phase_row);
            fwd_row_of<LOGN, CLASSES>(cls, smem + j * N, tau, m, false);
        }
        phase_row ^= 1;
        // ---- tensor step
        __syncthreads();
        cluster_arrive();  // this CTA's two rows are final
        const int64_t comp = (int64_t)R * N;  // words between the components of ten
        u64 *out = ten + ((int64_t)3 * item * R + r) * N;
        if (has_class(CLASSES, kNarrowH) && cls == kNarrowH) tensor_step<LOGN, true>(smem, smem + N, out, comp, rank, tau, S.p, S.ninv);
        else tensor_step<LOGN, false>(smem, smem + N, out, comp, rank, tau, S.p, S.ninv);
        // the generic-proxy accesses to these buffers come before their next TMA refill
        fence_proxy_async_smem();
        cluster_arrive_relaxed();  // this CTA has finished reading the peer's rows (waited for before the next refill / exit)
    }
    if (first < tasks) cluster_wait();  // the peer may still be reading this CTA's rows
}

// ---------------------------------------------------------------------------------------------- launch
static void build_row_list(const Context &ctx, const NttRowMap &map, bool inverse, RowList &rl) {
    rl.rows_per_poly = map.rows_per_poly;
    rl.count = 0;
    rl.src_poly_stride = map.src_mod ? map.src_poly_stride : (long long)map.rows_per_poly * ctx.n;
    // class-major order (the cheapest rows last, so the tail of the launch is made of short rows)
    static const int order[5] = {kWide, kMid, kNarrow, kNarrowH, kSmall};
    for (int oi = 0; oi < 5; ++oi) {
        const int cls = order[oi];
        for (int r = 0; r < map.rows_per_poly; ++r) {
            const int slot = map.slot[r / map.group];
            if (class_of_modulus(ctx.slots[slot].dev.p, ctx.slots[slot].dev.bits) != cls) continue;
            const int i = rl.count++;
            rl.row[i] = (unsigned short)r;
            rl.slot[i] = (unsigned short)slot;
            rl.src_row[i] = (unsigned short)(map.src_mod && !inverse ? r % map.src_mod : r);
            int flags = cls;
            if (map.src_mod && !inverse) {
                // inputs are residues mod the source modulus: fine as they are while they stay inside the lazy input
                // range of the butterflies (< 2p NARROW, < 8p MID, < 4p WIDE); otherwise re-reduce on load
                // (Bfv+Keys.swift:168-172)
                const u64 p = ctx.slots[slot].dev.p, src_p = ctx.slots[map.src_slot[r % map.src_mod]].dev.p;
                const u64 room = narrow_like(cls) ? 2u : cls == kMid ? 8u : cls == kSmall ? 1u : 4u;
                if (src_p > p && (src_p - 1) / p >= room) flags |= 8;
            }
            rl.flags[i] = (unsigned char)flags;
        }
    }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}
// 2-D view of a u64 buffer for the row copies: dimension 0 = the 16 words of a 128-byte line, dimension 1 = lines
static bool make_line_map(CUtensorMap *map, const u64 *base, int logn) {
    EncodeTiledFn enc = encode_tiled();
    if (!enc || (reinterpret_cast<uintptr_t>(base) & 15)) return false;
    const int lines = (1 << logn) / kLineWords;
    const cuuint64_t dims[2] = {kLineWords, (cuuint64_t)1 << 31};  // extent only bounds the coordinates
    const cuuint64_t strides[1] = {kLineWords * sizeof(u64)};
    const cuuint32_t box[2] = {kLineWords, (cuuint32_t)(lines > kBoxLines ? kBoxLines : lines)};
    const cuuint32_t elem_strides[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<u64 *>(base), dims, strides, box, elem_strides,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Whether a launch has NARROW-H rows and every other row is NARROW: at N = 2^13 such launches (the multiply's [Q, aux]
// rows) run the kernels compiled for kNarrowClasses.  Launches of NARROW rows alone keep the all-class kernels: the
// two-class kernel measured 0.5-0.9 % slower on them (C2 with plain auxiliary primes, C1-8192; DESIGN.md section 4).
// Other sizes have the all-class kernels only.
static bool narrow_h_rows(const RowList &rl) {
    bool any_h = false;
    for (int i = 0; i < rl.count; ++i) {
        const int cls = rl.flags[i] & 7;
        if (!narrow_like(cls)) return false;
        any_h |= cls == kNarrowH;
    }
    return any_h;
}

template <int LOGN, bool INVERSE, unsigned CLASSES>
static cudaError_t launch_rows(const Context &ctx, const RowList &rl, const u64 *in, u64 *out, int polys, int64_t rows,
                               int scale_mode, cudaStream_t stream) {
    CUtensorMap map_in, map_out;
    if (!make_line_map(&map_in, in, LOGN) || !make_line_map(&map_out, out, LOGN)) return cudaErrorInvalidValue;
    constexpr int threads = (1 << LOGN) / 16;
    constexpr size_t smem = ntt_smem_bytes<LOGN>();
    auto k = ntt_rows_kernel<LOGN, INVERSE, CLASSES>;
    static int ctas_per_sm[64] = {0};  // per instantiation and device
    static std::mutex mu;
    int per_sm;
    {
        std::lock_guard<std::mutex> lock(mu);
        int &c = ctas_per_sm[ctx.device & 63];
        if (c == 0) {
            cudaError_t e;
            if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
            int n = 0;
            if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k, threads, smem)) != cudaSuccess) return e;
            if (n < 1) return cudaErrorInvalidConfiguration;
            c = n;
        }
        per_sm = c;
    }
    const int64_t grid = std::min<int64_t>(rows, (int64_t)ctx.sm_count * per_sm);
    ++g_kernel_launches;
    k<<<(unsigned)grid, threads, smem, stream>>>(map_in, map_out, ctx.d_slots, rl, polys, scale_mode);
    return cudaGetLastError();
}

template <int LOGN, bool INVERSE>
static cudaError_t launch_logn(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               int scale_mode, cudaStream_t stream) {
    if (rows % map.rows_per_poly) return cudaErrorInvalidValue;
    if (rows == 0) return cudaSuccess;
    if (rows > 0x7fffffffLL) return cudaErrorInvalidValue;
    RowList rl;
    build_row_list(ctx, map, INVERSE, rl);
    if (rl.src_poly_stride % kLineWords) return cudaErrorInvalidValue;
    const int polys = (int)(rows / map.rows_per_poly);
    if (LOGN == 13 && narrow_h_rows(rl))
        return launch_rows<LOGN, INVERSE, (LOGN == 13 ? kNarrowClasses : kAllClasses)>(ctx, rl, in, out, polys, rows, scale_mode, stream);
    return launch_rows<LOGN, INVERSE, kAllClasses>(ctx, rl, in, out, polys, rows, scale_mode, stream);
}

// ---------------------------------------------------------------------------------------------- N = 2^15
// A 2^15 row (256 KB) does not fit one CTA's shared memory.  Its first forward stage (pairs i, i + N/2, one twiddle) and
// last inverse stage are elementwise over the two halves; in between each half is an independent 2^14-point transform
// that uses the entries (2 + h) 2^s + g of the twiddle table, which context.cu lays out as a table of its own ("virtual
// slot").  So: forward = split kernel (global memory, also performs the key-switch gather) + the 2^14 kernel over twice
// as many rows; inverse = the 2^14 kernel with the `partial` flag + merge kernel (N^-1 scaling).
struct SplitRows {
    int rows_per_poly, count;
    unsigned short row[kMaxRowList];
    unsigned short src_row[kMaxRowList], slot[kMaxRowList];
    unsigned char reduce_in[kMaxRowList];
    long long src_poly_stride;
};
__global__ void __launch_bounds__(256) ntt_split_forward_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                               const ModSlot *__restrict__ slots,
                                                               const __grid_constant__ SplitRows sr, int polys, int logn) {
    const int64_t n = (int64_t)1 << logn, half = n >> 1;
    const int which = blockIdx.y;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;  // two adjacent coefficients per thread
    if (i >= half) return;
    const ModSlot &S = slots[sr.slot[which]];
    const u64 p = S.p;
    const ulonglong2 w = S.tw[1];
    for (int64_t poly = blockIdx.z; poly < polys; poly += gridDim.z) {  // grid z is capped at 65535
        const u64 *src = in + poly * sr.src_poly_stride + ((int64_t)sr.src_row[which] << logn) + i;
        u64 *dst = out + (((poly * sr.rows_per_poly) + sr.row[which]) << logn) + i;
        ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(src), y = *reinterpret_cast<const ulonglong2 *>(src + half);
        if (sr.reduce_in[which]) {  // gathered key-switch digit: residues of another modulus (Bfv+Keys.swift:168-172)
            x.x = barrett64(x.x, p, S.mu1), x.y = barrett64(x.y, p, S.mu1);
            y.x = barrett64(y.x, p, S.mu1), y.y = barrett64(y.y, p, S.mu1);
        }
        const u64 v0 = shoup_mul(y.x, w.x, w.y, p), v1 = shoup_mul(y.y, w.x, w.y, p);
        *reinterpret_cast<ulonglong2 *>(dst) = make_ulonglong2(add_mod(x.x, v0, p), add_mod(x.y, v1, p));
        *reinterpret_cast<ulonglong2 *>(dst + half) = make_ulonglong2(sub_mod(x.x, v0, p), sub_mod(x.y, v1, p));
    }
}
__global__ void __launch_bounds__(256) ntt_merge_inverse_kernel(u64 *__restrict__ data, const ModSlot *__restrict__ slots,
                                                               const __grid_constant__ SplitRows sr, int polys, int logn,
                                                               int scale_mode) {
    const int64_t n = (int64_t)1 << logn, half = n >> 1;
    const int which = blockIdx.y;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (i >= half) return;
    const ModSlot &S = slots[sr.slot[which]];
    const u64 p = S.p;
    const ModSlot::InvScale sc = S.inv_scale[scale_mode];
    for (int64_t poly = blockIdx.z; poly < polys; poly += gridDim.z) {  // grid z is capped at 65535
        u64 *row = data + (((poly * sr.rows_per_poly) + sr.row[which]) << logn) + i;
        const ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(row), y = *reinterpret_cast<const ulonglong2 *>(row + half);
        // (x + y) N^-1 and (x - y) N^-1 psi^-(N/2), each times the scaling of scale_mode (PolyRq+Ntt.swift:416-419)
        *reinterpret_cast<ulonglong2 *>(row) =
            make_ulonglong2(shoup_mul(x.x + y.x, sc.c0, sc.c0p, p), shoup_mul(x.y + y.y, sc.c0, sc.c0p, p));
        *reinterpret_cast<ulonglong2 *>(row + half) =
            make_ulonglong2(shoup_mul(x.x - y.x + p, sc.c1, sc.c1p, p), shoup_mul(x.y - y.y + p, sc.c1, sc.c1p, p));
    }
}

template <bool INVERSE>
static cudaError_t launch_split(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows, int scale_mode,
                                cudaStream_t stream) {
    constexpr int LOGN = kMaxLogN;  // the half transforms
    if (rows % map.rows_per_poly) return cudaErrorInvalidValue;
    if (rows == 0) return cudaSuccess;
    if (rows * 2 > 0x7fffffffLL || 2 * map.rows_per_poly > kMaxRowList) return cudaErrorInvalidValue;
    const int polys = (int)(rows / map.rows_per_poly);
    RowList full;
    build_row_list(ctx, map, INVERSE, full);
    SplitRows sr;
    sr.rows_per_poly = full.rows_per_poly;
    sr.count = full.count;
    sr.src_poly_stride = full.src_poly_stride;
    RowList rl;  // the half rows: row 2r + h of a polynomial with twice as many rows, on the virtual slot of (slot, h)
    rl.rows_per_poly = 2 * full.rows_per_poly;
    rl.count = 2 * full.count;
    rl.src_poly_stride = (long long)rl.rows_per_poly << LOGN;
    for (int i = 0; i < full.count; ++i) {
        sr.row[i] = full.row[i];
        sr.slot[i] = full.slot[i];
        sr.src_row[i] = full.src_row[i];
        // any gathered row is re-reduced here (cheap next to the two transforms), so the halves see canonical residues
        sr.reduce_in[i] = (unsigned char)((map.src_mod && !INVERSE) ? 1 : 0);
        for (int hh = 0; hh < 2; ++hh) {
            const int j = 2 * i + hh;
            rl.row[j] = (unsigned short)(2 * full.row[i] + hh);
            rl.src_row[j] = rl.row[j];  // the half transforms run in place: source row = the row itself
            rl.slot[j] = (unsigned short)(ctx.split_slot_base + 2 * full.slot[i] + hh);
            rl.flags[j] = (unsigned char)((full.flags[i] & 7) | (INVERSE ? 16 : 0));
        }
    }
    // the split and merge kernels loop over the polynomials past grid z's limit
    const dim3 egrid((unsigned)((ctx.n / 4 + 255) / 256), (unsigned)full.count, (unsigned)std::min(polys, 65535));
    if (!INVERSE) {
        ++g_kernel_launches;
        ntt_split_forward_kernel<<<egrid, 256, 0, stream>>>(in, out, ctx.d_slots, sr, polys, ctx.logn);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        in = out;
    }
    // the 2^14 kernel over the 2 x rows half rows, in place over `out` (forward) / from `in` to `out` (inverse); rows
    // addressed like inverse rows
    cudaError_t e = launch_rows<LOGN, INVERSE, kAllClasses>(ctx, rl, in, out, polys, 2 * rows, scale_mode, stream);
    if (e != cudaSuccess) return e;
    if (INVERSE) {
        ++g_kernel_launches;
        ntt_merge_inverse_kernel<<<egrid, 256, 0, stream>>>(out, ctx.d_slots, sr, polys, ctx.logn, scale_mode);
        return cudaGetLastError();
    }
    return cudaSuccess;
}

bool ntt_fast_supported(const Context &ctx) { return ctx.logn >= kMinLogN && ctx.logn <= kSplitLogN; }

template <bool INVERSE>
static cudaError_t launch_fast(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               int scale_mode, cudaStream_t stream) {
    switch (ctx.logn) {
        case 10: return launch_logn<10, INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        case 11: return launch_logn<11, INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        case 12: return launch_logn<12, INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        case 13: return launch_logn<13, INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        case 14: return launch_logn<14, INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        case 15: return launch_split<INVERSE>(ctx, map, in, out, rows, scale_mode, stream);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_ntt_forward_fast(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                    cudaStream_t stream) {
    return launch_fast<false>(ctx, map, in, out, rows, 0, stream);
}
cudaError_t launch_ntt_inverse_fast(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                                    int scale_mode, cudaStream_t stream) {
    return launch_fast<true>(ctx, map, in, out, rows, scale_mode, stream);
}

template <unsigned CLASSES>
static cudaError_t launch_forward_tensor(const Context &ctx, const RowList &rl, const u64 *lhs, const u64 *rhs,
                                         const u64 *ext, u64 *ten, int64_t items, cudaStream_t stream) {
    constexpr int LOGN = 13;
    CUtensorMap map_lhs, map_rhs, map_ext;
    if (!make_line_map(&map_lhs, lhs, LOGN) || !make_line_map(&map_rhs, rhs, LOGN) || !make_line_map(&map_ext, ext, LOGN))
        return cudaErrorInvalidValue;
    constexpr int threads = (1 << LOGN) / 16;
    constexpr size_t smem = ntt_tensor_smem_bytes<LOGN>();
    auto k = ntt_forward_tensor_kernel<LOGN, CLASSES>;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    static int clusters_per_device[64] = {0};  // clusters of two CTAs the device holds at once
    static std::mutex mu;
    int clusters;
    {
        std::lock_guard<std::mutex> lock(mu);
        int &c = clusters_per_device[ctx.device & 63];
        if (c == 0) {
            cudaError_t e;
            if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
            cfg.gridDim = dim3(2 * ctx.sm_count);
            int n = 0;
            if ((e = cudaOccupancyMaxActiveClusters(&n, k, &cfg)) != cudaSuccess) return e;
            if (n < 1) return cudaErrorInvalidConfiguration;
            c = n;
        }
        clusters = c;
    }
    const int64_t tasks = items * rl.count;
    cfg.gridDim = dim3((unsigned)(2 * std::min<int64_t>(tasks, clusters)));
    ++g_kernel_launches;
    cudaError_t e = cudaLaunchKernelEx(&cfg, k, map_lhs, map_rhs, map_ext, ten, (const ModSlot *)ctx.d_slots, rl, (int)items, ctx.L);
    return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t launch_ntt_forward_tensor(const Context &ctx, const NttRowMap &map, const u64 *lhs, const u64 *rhs,
                                      const u64 *ext, u64 *ten, int64_t items, cudaStream_t stream) {
    if (ctx.logn != 13) return cudaErrorInvalidValue;
    if (items == 0) return cudaSuccess;
    // every line index of ext (the largest buffer read) fits an int
    if (items * 4 * map.rows_per_poly * (ctx.n / kLineWords) > 0x7fffffffLL) return cudaErrorInvalidValue;
    RowList rl;
    build_row_list(ctx, map, false, rl);
    if (narrow_h_rows(rl)) return launch_forward_tensor<kNarrowClasses>(ctx, rl, lhs, rhs, ext, ten, items, stream);
    return launch_forward_tensor<kAllClasses>(ctx, rl, lhs, rhs, ext, ten, items, stream);
}

}  // namespace hecuda
