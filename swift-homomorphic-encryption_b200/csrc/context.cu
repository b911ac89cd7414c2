// context.cu -- builds the immutable device context (see context.hpp for the reference mapping).
#include "context.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "hostmath.hpp"
#include "ntt_fast.cuh"

namespace hecuda {
using namespace host;


static void fill_barrett(u64 p, u64 &mu1, u64 &mu_hi, u64 &mu_lo) {
    mu1 = (u64)(((u128)1 << 64) / p);
    u128 mu = (p & (p - 1)) == 0 ? ((u128)1 << (128 - (bit_length(p) - 1))) : (~(u128)0) / p;
    mu_hi = (u64)(mu >> 64);
    mu_lo = (u64)mu;
}

// floor_w: the extra factor of kScaleTMontFloor ((Q/q_i)^-1 mod q_i on a ciphertext modulus, 1 elsewhere)
static bool build_slot(HostSlot &hs, u64 p, int64_t n, int logn, u64 t, u64 floor_w, std::vector<ulonglong2> &tw,
                       std::vector<ulonglong2> &itw, std::string &err) {
    if (!is_prime(p) || (p - 1) % (2 * (u64)n) != 0) {
        err = "invalidNttModulus: " + std::to_string(p) + " is not a prime = 1 mod 2N";
        return false;
    }
    if (p >= (1ull << 62)) {  // Modulus<UInt64>.max, Sources/ModularArithmetic/Modulus.swift:177-180
        err = "invalidModulus: " + std::to_string(p) + " exceeds 2^62 - 1";
        return false;
    }
    ModSlot &d = hs.dev;
    std::memset(&d, 0, sizeof(d));
    d.p = p;
    fill_barrett(p, d.mu1, d.mu_hi, d.mu_lo);
    d.bits = bit_length(p);
    d.s_prod = d.bits - 2;
    d.mu_prod = (u64)(((u128)1 << (d.bits + 62)) / p);
    d.red_shift = d.bits > 12 ? d.bits - 12 : 0;
    d.red_recip = (u32)((((u128)1) << (d.red_shift + 32)) / p);
    const u64 psi = min_primitive_root(2 * (u64)n, p);
    const u64 psi_inv = invmod(psi, p);
    hs.roots.assign(n, 1);
    hs.inv_roots.assign(n, 1);
    // roots[bitrev(i)] = psi^i   (PolyRq+Ntt.swift:125-137); inverse table uses the same indexing here.
    u64 pw = 1, ipw = 1;
    for (int64_t i = 0; i < n; ++i) {
        unsigned r = bitrev((unsigned)i, logn);
        hs.roots[r] = pw;
        hs.inv_roots[r] = ipw;
        pw = mulmod(pw, psi, p);
        ipw = mulmod(ipw, psi_inv, p);
    }
    tw.resize(n);
    itw.resize(n);
    for (int64_t i = 0; i < n; ++i) {
        tw[i] = make_ulonglong2(hs.roots[i], shoup_factor(hs.roots[i], p));
        itw[i] = make_ulonglong2(hs.inv_roots[i], shoup_factor(hs.inv_roots[i], p));
    }
    const u64 n_inv = invmod((u64)n % p, p);
    const u64 w1_inv = n > 1 ? hs.inv_roots[1] : 1;  // psi^-(N/2)
    d.r64 = (u64)(((u128)1 << 64) % p);
    {   // -p^-1 mod 2^64 by Newton iteration
        u64 inv = p;  // correct to 3 bits for odd p
        for (int i = 0; i < 6; ++i) inv *= 2 - p * inv;
        d.ninv = 0 - inv;
    }
    const u64 scalings[4] = {1 % p, mulmod(t % p, d.r64, p), d.r64, mulmod(mulmod(t % p, d.r64, p), floor_w % p, p)};
    for (int k = 0; k < 4; ++k) {
        ModSlot::InvScale &sc = d.inv_scale[k];
        sc.c0 = mulmod(n_inv, scalings[k], p);
        sc.c0p = shoup_factor(sc.c0, p);
        sc.c1 = mulmod(sc.c0, w1_inv, p);
        sc.c1p = shoup_factor(sc.c1, p);
    }
    return true;
}

static DivRoundConsts build_divround(const std::vector<u64> &base) {
    DivRoundConsts c;
    std::memset(&c, 0, sizeof(c));
    c.l = (int)base.size();
    c.last = base.back();
    c.half = c.last >> 1;
    for (int i = 0; i + 1 < c.l; ++i) {
        const u64 m = base[i];
        c.m[i] = m;
        c.mu1[i] = (u64)(((u128)1 << 64) / m);
        c.half_mod[i] = c.half % m;
        c.inv_w[i] = invmod(c.last % m, m);
        c.inv_wp[i] = shoup_factor(c.inv_w[i], m);
    }
    return c;
}

// PolyContext.maxLazyProductAccumulationCount (PolyContext.swift:246-253): the largest count of products
// (q_max - 1)^2 that, added to q_max, stays within the double word of the scalar type
static int64_t max_lazy_product_count(u64 qmax, int word_bits) {
    if (qmax < 2) return INT64_MAX;
    const u128 double_max = word_bits == 64 ? ~(u128)0 : (u128)~(u64)0;
    const u128 count = (double_max - qmax) / ((u128)(qmax - 1) * (qmax - 1));
    return count > (u128)INT64_MAX ? INT64_MAX : (int64_t)count;
}

Context *Context::create(int64_t n, const u64 *coeff_moduli, int nmod, u64 t, std::string &err, int word_bits) {
    if (word_bits != 64 && word_bits != 32) { err = "invalidEncryptionParameters: word size must be 32 or 64"; return nullptr; }
    for (int i = 0; i < nmod; ++i)  // Modulus<T>.max = 2^(bitWidth - 2) - 1, Sources/ModularArithmetic/Modulus.swift:177-180
        if (coeff_moduli[i] >> (word_bits - 2)) { err = "invalidModulus: " + std::to_string(coeff_moduli[i]) + " exceeds the maximum of this word size"; return nullptr; }
    if (n < 2 || (n & (n - 1)) || n > (1 << 17)) { err = "invalidDegree: N must be a power of two in [2, 2^17]"; return nullptr; }
    // the NTT kernels keep a whole row in one CTA's shared memory: N <= 2^14 (a 2^15 row is 256 KB)
    // 2^15 (the reference's largest predefined degree, EncryptionParameters.swift:199-206) runs as one cross-half stage
    // plus two 2^14 transforms (ntt_fast.cu)
    if (n > (1 << fast::kSplitLogN)) { err = "unsupportedHeOperation: polynomial degrees above 2^" + std::to_string(fast::kSplitLogN) + " are not supported by the NTT kernels"; return nullptr; }
    if (nmod < 1) { err = "invalidEncryptionParameters: need at least one coefficient modulus"; return nullptr; }
    if (nmod > kMaxL) { err = "invalidEncryptionParameters: more than " + std::to_string(kMaxL) + " coefficient moduli (EncryptionParameters.swift:148)"; return nullptr; }
    if (t < 2) { err = "invalidEncryptionParameters: plaintext modulus"; return nullptr; }
    for (int i = 0; i < nmod; ++i)
        for (int j = 0; j < i; ++j)
            if (coeff_moduli[i] == coeff_moduli[j]) { err = "coprimeModuli: repeated coefficient modulus"; return nullptr; }
    if (nmod >= 2) {  // the largest key-switching context holds every modulus (Context.swift:114-124)
        u64 qmax = 0;
        for (int i = 0; i < nmod; ++i) qmax = coeff_moduli[i] > qmax ? coeff_moduli[i] : qmax;
        if (nmod >= max_lazy_product_count(qmax, word_bits)) {
            err = "invalidEncryptionParameters: " + std::to_string(nmod) + " moduli reach maxLazyProductAccumulationCount of the key-switching context";
            return nullptr;
        }
    }

    Context *c = new Context();
    c->n = n;
    c->logn = bit_length((u64)n) - 1;
    // one coefficient modulus: it is the ciphertext modulus and there is no key-switching modulus (Context.swift:102-107)
    c->has_ks = nmod >= 2;
    c->L = c->has_ks ? nmod - 1 : 1;
    c->t = t;
    c->word_bits = word_bits;
    c->mtilde = word_bits == 64 ? (1ull << 32) : (1ull << 16);                       // Scalar.swift:509-511, 522-524
    c->gamma = word_bits == 64 ? ((1ull << 62) - 40797) : ((1ull << 30) - 20405);    // Scalar.swift:503-507, 516-520
    const u64 kMTilde = c->mtilde;
    cudaGetDevice(&c->device);
    c->sm_count = 1;
    cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, c->device);
    const int L = c->L;
    c->q.assign(coeff_moduli, coeff_moduli + L);
    c->q_ks = c->has_ks ? coeff_moduli[L] : 0;
    for (u64 qi : c->q)
        if (t >= qi) { err = "invalidEncryptionParameters: plaintext modulus must be below every coefficient modulus"; delete c; return nullptr; }
    // BEHZ auxiliary base: the L+1 smallest (bitWidth - 3)-bit NTT primes (RnsTool.swift:30-33)
    c->bsk = smallest_ntt_primes(word_bits - 3, L + 1, (u64)n);
    if ((int)c->bsk.size() != L + 1) { err = "notEnoughPrimes for Bsk"; delete c; return nullptr; }
    for (u64 b : c->bsk)
        for (int i = 0; i < nmod; ++i)
            if (b == coeff_moduli[i]) { err = "coprimeModuli: coefficient modulus collides with the BEHZ base"; delete c; return nullptr; }

    // ---- the auxiliary base the fused multiply computes in.  What Bfv.mulAssign returns does not depend on which
    // auxiliary primes BEHZ uses, as long as they are large enough for its exactness conditions: the lifted
    // operands y = (x~ + q r_m~) / m~, the tensor product D = y1 * y2 and F = floor(t D / q) - u (u = the overflow of the
    // fast base conversion of [t D]_q, a function of the q residues alone) are fixed integers, and the
    // Shenoy-Kumaresan conversion back to q is exact (RnsTool.swift:324-456).  So the multiply runs over L + 1 primes
    // below 2^55, whose NTT rows never need a conditional subtraction (ntt_fast.cuh, NARROW class), instead of the
    // reference's 61-bit Bsk; the reference base stays available for the stage-level entry points.  The 55-bit primes
    // are the smallest of the form h 2^32 + 1: their butterflies (NARROW-H) and Montgomery reductions (mont_reduce_h)
    // need fewer multiplies.  Conditions checked, each with one bit to spare in the log2 test below:
    //   q * B_aux > 8 N q^2   (D is represented exactly),   B_aux(L primes) * m_sk > 16 t N q   (F survives SK)
    // They bound ONE tensor product.  The ct x ct inner product floors the sum of `pairs` products once, so D and F
    // grow by that factor: aux_max_pairs is the largest P for which both still hold with log2(P) added to their right-hand
    // sides, and longer inner products run over Bsk instead (capi.cu inner_product_chunk).
    c->aux = c->bsk;
    {
        const char *env = std::getenv("HECUDA_AUX_BASE");
        const bool want_fast = !(env && std::string(env) == "reference");
        // cheapest NTT class first: primes below 2^30 (32-bit butterflies) when q is small enough for them, else below 2^55
        const int widths[2] = {30, 55};
        double log_q = 0;
        for (u64 v : c->q) log_q += std::log2((double)v);
        const double log_n = (double)c->logn, log_t = std::log2((double)t);
        for (int wi = 0; wi < 2 && want_fast && c->aux == c->bsk && word_bits == 64; ++wi) {
            // 55 bits: primes = 1 mod 2^32 (NTT-friendly for every supported N)
            std::vector<u64> cand = widths[wi] == 55 ? smallest_ntt_primes(55, L + 1 + nmod, 1ull << 31)
                                                     : smallest_ntt_primes(widths[wi], L + 1 + nmod, (u64)n);
            std::vector<u64> pick;
            for (u64 v : cand) {
                bool used = false;
                for (int i = 0; i < nmod; ++i) used |= coeff_moduli[i] == v;
                if (!used && (int)pick.size() < L + 1) pick.push_back(v);
            }
            double log_aux = 0, log_aux_l = 0;
            for (size_t j = 0; j < pick.size(); ++j) {
                log_aux += std::log2((double)pick[j]);
                if ((int)j < L) log_aux_l += std::log2((double)pick[j]);
            }
            if ((int)pick.size() != L + 1) continue;
            const double slack_d = log_aux - (log_q + log_n + 4);
            const double slack_f = log_aux_l + std::log2((double)pick.back()) - (log_t + log_n + log_q + 5);
            const double slack = std::min(slack_d, slack_f);
            if (slack >= 0) {
                c->aux = pick;
                c->aux_max_pairs = slack >= 62 ? INT64_MAX : (int64_t)std::floor(std::exp2(slack));
            }
        }
    }
    c->aux_is_reference = c->aux == c->bsk;

    // ---- NTT slots.  The plaintext modulus gets one when it is NTT-friendly (SIMD encoding, Encoding.swift:197-201), after
    // every other slot so that the ciphertext-side slot indices do not depend on t.
    c->simd = is_prime(t) && (t - 1) % (2 * (u64)n) == 0;
    const int nslots = (c->aux_is_reference ? 2 * L + 2 : 3 * L + 3) + (c->simd ? 1 : 0);
    c->slots.resize(nslots);
    std::vector<u64> slot_mod(nslots);
    if (c->simd) slot_mod[c->slot_t()] = t;
    for (int i = 0; i < L; ++i) slot_mod[c->slot_q(i)] = c->q[i];
    for (int j = 0; j <= L; ++j) slot_mod[c->slot_bsk(j)] = c->bsk[j];
    slot_mod[c->slot_ks()] = c->q_ks;
    if (!c->aux_is_reference)
        for (int j = 0; j <= L; ++j) slot_mod[c->slot_aux(j)] = c->aux[j];
    const size_t table_bytes = sizeof(ulonglong2) * (size_t)n;
    const bool fast = c->logn >= fast::kMinLogN && c->logn <= fast::kMaxLogN;
    const bool split = c->logn == fast::kSplitLogN;  // two half-size transforms per row, each with its own twiddle view
    const int half_logn = c->logn - 1;
    const int64_t half_n = n / 2;
    const int threads = (int)((split ? half_n : n) / 16);
    // N = 2^13: the resident twiddle images instead of the transposed tables (ntt_fast.cuh)
    const bool resident = fast && fast::resident_twiddles(c->logn);
    const size_t tr_bytes = (fast || split) && !resident ? sizeof(ulonglong2) * (size_t)15 * threads : 0;  // transposed line-owning-pass tables
    const size_t img_bytes = resident ? sizeof(ulonglong2) * (size_t)fast::image_entries(c->logn) : 0;
    const size_t half_bytes = sizeof(ulonglong2) * (size_t)half_n;
    // per slot: [tw][itw] then, unsplit: [tw_t][itw_t] or [tw_img][itw_img]; split: per half [tw_h][itw_h][tw_t_h][itw_t_h]
    const size_t slot_bytes = 2 * table_bytes + (split ? 2 * (2 * half_bytes + 2 * tr_bytes) : 2 * tr_bytes + 2 * img_bytes);
    if (cudaMalloc(&c->d_pool, slot_bytes * nslots) != cudaSuccess) { err = "cudaMalloc failed for twiddle tables"; delete c; return nullptr; }
    std::vector<ulonglong2> tw, itw, tr(15 * (size_t)threads), itr(15 * (size_t)threads), twh, itwh;
    std::vector<ModSlot> dev_slots(split ? 3 * nslots : nslots);
    c->split_slot_base = split ? nslots : 0;
    for (int s = 0; s < nslots; ++s) {
        if (s == c->slot_ks() && !c->has_ks) {  // no key-switching modulus: the slot stays empty
            std::memset(&c->slots[s].dev, 0, sizeof(ModSlot));
            dev_slots[s] = c->slots[s].dev;
            continue;
        }
        const u64 floor_w = s < L ? invmod(punctured_mod(c->q.data(), L, s, slot_mod[s]), slot_mod[s]) : 1;  // slot_q(i) = i
        if (!build_slot(c->slots[s], slot_mod[s], n, c->logn, t, floor_w, tw, itw, err)) { delete c; return nullptr; }
        char *base = (char *)c->d_pool + slot_bytes * s;
        cudaMemcpy(base, tw.data(), table_bytes, cudaMemcpyHostToDevice);
        cudaMemcpy(base + table_bytes, itw.data(), table_bytes, cudaMemcpyHostToDevice);
        c->slots[s].dev.tw = (const ulonglong2 *)base;
        c->slots[s].dev.itw = (const ulonglong2 *)(base + table_bytes);
        if (resident) {
            // the image keeps the even groups of the stage with N/2 twiddles only: check w_i = w_(i-1) zeta for every odd
            // i there, zeta = psi^(N/2) = tw[1] (inverse psi^(-N/2) = itw[1])
            const u64 p = slot_mod[s];
            for (int64_t i = n / 2 + 1; i < n; i += 2)
                if (tw[i].x != mulmod(tw[i - 1].x, tw[1].x, p) || itw[i].x != mulmod(itw[i - 1].x, itw[1].x, p)) {
                    err = "internal error: twiddle table of " + std::to_string(p) + " is not in bit-reversed order";
                    delete c;
                    return nullptr;
                }
            const int entries = fast::image_entries(c->logn);
            std::vector<ulonglong2> img(entries), iimg(entries);
            for (int i = 0; i < entries; ++i) {
                img[i] = tw[fast::image_source(c->logn, false, i)];
                iimg[i] = itw[fast::image_source(c->logn, true, i)];
            }
            cudaMemcpy(base + 2 * table_bytes, img.data(), img_bytes, cudaMemcpyHostToDevice);
            cudaMemcpy(base + 2 * table_bytes + img_bytes, iimg.data(), img_bytes, cudaMemcpyHostToDevice);
            c->slots[s].dev.tw_img = (const ulonglong2 *)(base + 2 * table_bytes);
            c->slots[s].dev.itw_img = (const ulonglong2 *)(base + 2 * table_bytes + img_bytes);
        } else if (fast) {
            for (int k = 0; k < 15; ++k)
                for (int tau = 0; tau < threads; ++tau) {
                    tr[(size_t)k * threads + tau] = tw[fast::fwd_last_source(c->logn, k, tau)];
                    itr[(size_t)k * threads + tau] = itw[fast::inv_first_source(c->logn, k, tau)];
                }
            cudaMemcpy(base + 2 * table_bytes, tr.data(), tr_bytes, cudaMemcpyHostToDevice);
            cudaMemcpy(base + 2 * table_bytes + tr_bytes, itr.data(), tr_bytes, cudaMemcpyHostToDevice);
            c->slots[s].dev.tw_t = (const ulonglong2 *)(base + 2 * table_bytes);
            c->slots[s].dev.itw_t = (const ulonglong2 *)(base + 2 * table_bytes + tr_bytes);
        }
        dev_slots[s] = c->slots[s].dev;
        if (split) {
            // After the cross-half stage, half h of a row is a 2^14-point transform whose stage s' (2^s' groups) uses the
            // full table's entries (2 + h) 2^s' + group: lay those out like a table of a 2^14 transform, so the 2^14
            // kernels run on the halves unchanged (virtual slot nslots + 2 s + h).
            for (int hh = 0; hh < 2; ++hh) {
                twh.assign(half_n, tw[0]);
                itwh.assign(half_n, itw[0]);
                for (int64_t i = 1; i < half_n; ++i) {
                    const int sp = bit_length((u64)i) - 1;
                    const int64_t src = ((int64_t)(2 + hh) << sp) + (i - ((int64_t)1 << sp));
                    twh[i] = tw[src];
                    itwh[i] = itw[src];
                }
                for (int k = 0; k < 15; ++k)
                    for (int tau = 0; tau < threads; ++tau) {
                        tr[(size_t)k * threads + tau] = twh[fast::fwd_last_source(half_logn, k, tau)];
                        itr[(size_t)k * threads + tau] = itwh[fast::inv_first_source(half_logn, k, tau)];
                    }
                char *hb = base + 2 * table_bytes + hh * (2 * half_bytes + 2 * tr_bytes);
                cudaMemcpy(hb, twh.data(), half_bytes, cudaMemcpyHostToDevice);
                cudaMemcpy(hb + half_bytes, itwh.data(), half_bytes, cudaMemcpyHostToDevice);
                cudaMemcpy(hb + 2 * half_bytes, tr.data(), tr_bytes, cudaMemcpyHostToDevice);
                cudaMemcpy(hb + 2 * half_bytes + tr_bytes, itr.data(), tr_bytes, cudaMemcpyHostToDevice);
                ModSlot v = c->slots[s].dev;
                v.tw = (const ulonglong2 *)hb;
                v.itw = (const ulonglong2 *)(hb + half_bytes);
                v.tw_t = (const ulonglong2 *)(hb + 2 * half_bytes);
                v.itw_t = (const ulonglong2 *)(hb + 2 * half_bytes + tr_bytes);
                dev_slots[nslots + 2 * s + hh] = v;
            }
        }
    }
    if (cudaMalloc(&c->d_slots, sizeof(ModSlot) * dev_slots.size()) != cudaSuccess) { err = "cudaMalloc failed"; delete c; return nullptr; }
    cudaMemcpy(c->d_slots, dev_slots.data(), sizeof(ModSlot) * dev_slots.size(), cudaMemcpyHostToDevice);

    // ---- BEHZ constants (top level)
    const u64 *Q = c->q.data();
    auto build_behz = [&](const std::vector<u64> &base, bool reference_base, LiftConsts &lf, FloorConsts &fl) {
    const u64 *BSK = base.data();
    const u64 msk = base[L];
    auto slot_of = [&](int j) { return reference_base ? c->slot_bsk(j) : c->slot_aux(j); };
    std::memset(&lf, 0, sizeof(lf));
    lf.L = L;
    bool h_primes = true;  // reductions modulo every b_j can take mont_reduce_h
    for (int j = 0; j <= L; ++j) h_primes &= fast::class_of_modulus(BSK[j], bit_length(BSK[j])) == fast::kNarrowH;
    lf.h_primes = h_primes ? 1 : 0;
    {
        const u64 q_mod_mt = prod_mod(Q, L, kMTilde);
        lf.neg_inv_q_mt = (u32)((kMTilde - invmod(q_mod_mt, kMTilde)) % kMTilde);
    }
    for (int i = 0; i < L; ++i) {
        const u64 qi = Q[i];
        lf.q[i] = qi;
        const u64 inv_punct = invmod(punctured_mod(Q, L, i, qi), qi);
        lf.in_w[i] = mulmod(kMTilde % qi, inv_punct, qi);
        lf.in_wp[i] = shoup_factor(lf.in_w[i], qi);
        lf.punct_mt[i] = (u32)punctured_mod(Q, L, i, kMTilde);
    }
    lf.mt_mask = (u32)(kMTilde - 1);
    lf.mt_half = (u32)(kMTilde >> 1);
    for (int j = 0; j <= L; ++j) lf.neg_off[j] = ((kMTilde + BSK[j] - 1) / BSK[j]) * BSK[j] - kMTilde;
    for (int j = 0; j <= L; ++j) {
        const u64 bj = BSK[j];
        lf.b[j] = bj;
        lf.b_ninv[j] = c->slots[slot_of(j)].dev.ninv;
        const u64 r64 = c->slots[slot_of(j)].dev.r64;
        const u64 mt_inv = mulmod(invmod(kMTilde % bj, bj), r64, bj);  // m~^-1 2^64
        for (int i = 0; i < L; ++i) lf.mat[j][i] = mulmod(punctured_mod(Q, L, i, bj), mt_inv, bj);
        lf.qr[j] = mulmod(prod_mod(Q, L, bj), mt_inv, bj);
    }
    std::memset(&fl, 0, sizeof(fl));
    fl.L = L;
    fl.h_primes = lf.h_primes;
    const u64 b_mod_msk = prod_mod(BSK, L, msk);
    const u64 r64_msk = c->slots[slot_of(L)].dev.r64;
    const u64 b_inv_msk = mulmod(invmod(b_mod_msk, msk), r64_msk, msk);  // B^-1 2^64
    fl.a_msk = (msk - b_inv_msk) % msk;
    for (int i = 0; i < L; ++i) {
        const u64 qi = Q[i];
        fl.q[i] = qi;
        fl.q_ninv[i] = c->slots[c->slot_q(i)].dev.ninv;
        fl.q_mu1[i] = c->slots[c->slot_q(i)].dev.mu1;
        const u64 r64 = c->slots[c->slot_q(i)].dev.r64;
        fl.inq_w[i] = invmod(punctured_mod(Q, L, i, qi), qi);
        fl.inq_wp[i] = shoup_factor(fl.inq_w[i], qi);
        for (int k = 0; k < L; ++k) fl.omat[i][k] = mulmod(punctured_mod(BSK, L, k, qi), r64, qi);
        fl.b_mod_q[i] = mulmod(prod_mod(BSK, L, qi), r64, qi);
        fl.neg_b_mod_q[i] = (qi - fl.b_mod_q[i]) % qi;
    }
    for (int j = 0; j <= L; ++j) {
        const u64 bj = BSK[j];
        fl.b[j] = bj;
        fl.b_ninv[j] = c->slots[slot_of(j)].dev.ninv;
        fl.b_mu1[j] = (u64)(((u128)1 << 64) / bj);
        // Q^-1 2^64, times (B/b_j)^-1 on the rows whose f_j only feeds w_j = [f_j (B/b_j)^-1]_{b_j}
        u64 q_inv = mulmod(invmod(prod_mod(Q, L, bj), bj), c->slots[slot_of(j)].dev.r64, bj);
        if (j < L) q_inv = mulmod(q_inv, invmod(punctured_mod(BSK, L, j, bj), bj), bj);
        fl.fq[j] = q_inv;
        for (int i = 0; i < L; ++i) {
            const u64 v = mulmod(punctured_mod(Q, L, i, bj), q_inv, bj);
            fl.fmat[j][i] = (bj - v) % bj;
        }
    }
    for (int k = 0; k < L; ++k) fl.amat[k] = mulmod(punctured_mod(BSK, L, k, msk), b_inv_msk, msk);
    };
    build_behz(c->bsk, true, c->lift, c->floor);
    if (c->aux_is_reference) {
        c->lift_mul = c->lift;
        c->floor_mul = c->floor;
    } else {
        build_behz(c->aux, false, c->lift_mul, c->floor_mul);
    }

    // ---- ranges of the lazy sums (behz.cu).  The fast path ends the lift sums with one conditional subtraction
    // ((b_j^2 + L q_max b_j) / 2^64 < b_j  <=>  b_j + L q_max < 2^64) and alpha with three (< 8 m_sk); parameter sets with
    // many wide moduli take a Barrett reduction there instead.  Every 128-bit accumulator must stay below 2^128.
    auto check_ranges = [&](const std::vector<u64> &base, LiftConsts &lf, FloorConsts &fl) -> bool {
        u64 qmax = 0, bmax = 0;
        for (u64 v : c->q) qmax = v > qmax ? v : qmax;
        for (u64 v : base) bmax = v > bmax ? v : bmax;
        const double worst = std::log2((double)(L + 2)) + std::log2((double)qmax) + std::log2((double)bmax);
        if (worst >= 127.0) return false;
        // (b + L q_max < 2^64 also keeps f_msk < 2 m_sk and with it alpha < 8 m_sk for every supported L)
        const bool wide = (u128)bmax + (u128)L * qmax >= ((u128)1 << 64);
        lf.wide_sums = fl.wide_sums = wide ? 1 : 0;
        for (int j = 0; j <= L; ++j) lf.b_mu1[j] = (u64)(((u128)1 << 64) / base[j]);
        fl.msk_mu1 = (u64)(((u128)1 << 64) / base[L]);
        return true;
    };
    if (!check_ranges(c->bsk, c->lift, c->floor) || !check_ranges(c->aux, c->lift_mul, c->floor_mul)) {
        err = "unsupportedHeOperation: " + std::to_string(L) + " ciphertext moduli of this size overflow the 128-bit lazy sums";
        delete c;
        return nullptr;
    }

    {   // key switching accumulates l products of two residues in 128 bits (keyswitch.cu)
        u64 mmax = c->q_ks;
        for (u64 v : c->q) mmax = v > mmax ? v : mmax;
        if (std::log2((double)L) + 2 * std::log2((double)mmax) >= 128.0) {
            err = "unsupportedHeOperation: " + std::to_string(L) + " moduli of this size overflow the key-switching accumulator";
            delete c;
            return nullptr;
        }
    }

    // ---- plaintext translate constants per level (Bfv+Encrypt.swift:75-139 with getRnsTool(moduliCount: l))
    c->translate.resize(L + 1);
    for (int l = 1; l <= L; ++l) {
        TranslateConsts &tc = c->translate[l];
        std::memset(&tc, 0, sizeof(tc));
        tc.l = l;
        tc.t = t;
        tc.t_threshold = (t + 1) / 2;
        tc.q_mod_t = prod_mod(Q, l, t);
        tc.q_mod_t_p = shoup_factor(tc.q_mod_t, t);
        for (int i = 0; i < l; ++i) {
            const u64 qi = Q[i];
            tc.q[i] = qi;
            // Q_l = t floor(Q_l / t) + [Q_l]_t and Q_l = 0 mod q_i  ->  floor(Q_l / t) = -[Q_l]_t t^-1 mod q_i
            tc.delta[i] = mulmod((qi - tc.q_mod_t % qi) % qi, invmod(t % qi, qi), qi);
            tc.delta_p[i] = shoup_factor(tc.delta[i], qi);
        }
    }

    // ---- SIMD encoding permutation (generateEncodingMatrix, Encoding.swift:197-219; generator 3, Galois.swift:169-171)
    if (c->simd) {
        std::vector<int32_t> matrix(n), inverse(n);
        const u64 mask = 2 * (u64)n - 1;
        u64 g = 1;
        for (int64_t i = 0; i < n / 2; ++i) {
            matrix[i] = (int32_t)bitrev((unsigned)((g - 1) >> 1), c->logn);
            matrix[n / 2 + i] = (int32_t)bitrev((unsigned)((mask - g) >> 1), c->logn);
            g = (g * 3) & mask;
        }
        for (int64_t i = 0; i < n; ++i) inverse[matrix[i]] = (int32_t)i;
        if (cudaMalloc(&c->d_simd_matrix, sizeof(int32_t) * 2 * (size_t)n) != cudaSuccess) { err = "cudaMalloc failed"; delete c; return nullptr; }
        c->d_simd_inverse = c->d_simd_matrix + n;
        cudaMemcpy(c->d_simd_matrix, matrix.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice);
        cudaMemcpy(c->d_simd_inverse, inverse.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice);
    }

    // ---- divide-and-round constants
    c->ks_divround.resize(L + 1);
    c->ms_divround.resize(L + 1);
    for (int l = 1; l <= L; ++l) {
        std::vector<u64> base(c->q.begin(), c->q.begin() + l);
        if (l >= 2) c->ms_divround[l] = build_divround(base);
        if (!c->has_ks) continue;
        base.push_back(c->q_ks);
        c->ks_divround[l] = build_divround(base);
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { err = std::string("CUDA error during context setup: ") + cudaGetErrorString(e); delete c; return nullptr; }
    return c;
}

Context::~Context() {
    if (d_pool) cudaFree(d_pool);
    if (d_slots) cudaFree(d_slots);
    if (d_simd_matrix) cudaFree(d_simd_matrix);
}

NttRowMap Context::map_q(int rows) const {
    NttRowMap m;
    std::memset(&m, 0, sizeof(m));
    m.rows_per_poly = rows;
    m.group = 1;
    m.src_mod = 0;
    m.src_poly_stride = 0;
    for (int r = 0; r < rows; ++r) m.slot[r] = (unsigned char)slot_q(r);
    return m;
}
NttRowMap Context::map_qbsk() const {
    NttRowMap m;
    std::memset(&m, 0, sizeof(m));
    m.rows_per_poly = 2 * L + 1;
    m.group = 1;
    m.src_mod = 0;
    m.src_poly_stride = 0;
    for (int r = 0; r < L; ++r) m.slot[r] = (unsigned char)slot_q(r);
    for (int j = 0; j <= L; ++j) m.slot[L + j] = (unsigned char)slot_bsk(j);
    return m;
}
NttRowMap Context::map_qaux() const {
    NttRowMap m = map_qbsk();
    if (!aux_is_reference)
        for (int j = 0; j <= L; ++j) m.slot[L + j] = (unsigned char)slot_aux(j);
    return m;
}
NttRowMap Context::map_ks(int l) const {
    NttRowMap m;
    std::memset(&m, 0, sizeof(m));
    m.rows_per_poly = l + 1;
    m.group = 1;
    m.src_mod = 0;
    m.src_poly_stride = 0;
    for (int r = 0; r < l; ++r) m.slot[r] = (unsigned char)slot_q(r);
    m.slot[l] = (unsigned char)slot_ks();
    return m;
}
NttRowMap Context::map_single(int slot) const {
    NttRowMap m;
    std::memset(&m, 0, sizeof(m));
    m.rows_per_poly = 1;
    m.group = 1;
    m.src_mod = 0;
    m.src_poly_stride = 0;
    m.slot[0] = (unsigned char)slot;
    return m;
}
NttRowMap Context::map_ks_digits(int l, long long target_poly_stride) const {
    NttRowMap m = map_ks(l);
    m.rows_per_poly = (l + 1) * l;
    m.group = l;
    m.src_mod = l;
    m.src_poly_stride = target_poly_stride;
    for (int j = 0; j < l; ++j) m.src_slot[j] = (unsigned char)slot_q(j);
    return m;
}
int Context::find_slot(u64 modulus) const {
    for (size_t s = 0; s < slots.size(); ++s)
        if (slots[s].dev.p == modulus) return (int)s;
    return -1;
}

}  // namespace hecuda
