// keyswitch.cu -- hybrid key switching (alpha = 1) and modulus switching.
//
//   Bfv._computeKeySwitchingUpdate   Bfv/Bfv+Keys.swift:123-208
//   Bfv.relinearize                  Bfv/Bfv.swift:201-219
//   PolyRq.divideAndRoundQLast       PolyRq/PolyRq.swift:365-393
//   Bfv.modSwitchDown                Bfv/Bfv.swift:163-171
//
// Stage kernels (v1): digits -> forward NTT (ntt.cu) -> mac -> inverse NTT -> finish.
#include "kernels.cuh"

namespace hecuda {

// The digits dig[item][r][j] = NTT_{m_r}([target row j]_{m_r}) are produced by the forward NTT itself, which gathers
// the target rows on load (NttRowMap::src_mod; Bfv+Keys.swift:165-179) -- there is no separate digit kernel.

struct KsMacConsts {
    int l, K;
    u64 p[kMaxL + 1], ninv[kMaxL + 1];
};

// prod[item][comp][r][.] = [ sum_j dig[item][r][j][.] * key[j][comp][keyrow(r)][.] ]_{m_r} * 2^-64   (Bfv+Keys.swift:180-202)
// 128-bit lazy accumulation like the reference (:187-190), one Montgomery reduction; the 2^-64 is undone by the
// kScaleMont scaling of the inverse NTT that follows.  The sum is below l p^2, so its high word is below l p / 4 < 4p
// (context.cu keeps l below maxLazyProductAccumulationCount: l <= 14 at 62 bits, and l <= 31 at 61 bits and below).
// Montgomery's result is below high word + p, which at l >= 13 and 62 bits would pass 2^64; subtracting 2p 2^64 (a
// multiple of p) from a sum whose high word is >= 2p keeps it below 3p.
__device__ __forceinline__ u64 ks_reduce(u128 acc, u64 p, u64 ninv) {
    if ((u64)(acc >> 64) >= 2 * p) acc -= (u128)(2 * p) << 64;
    return csub(csub(mont_reduce(acc, p, ninv), 2 * p), p);
}

// CLIENT_KEYS: item i (counted from keys.item0) uses keys.key[i / keys.items_per_client] instead of `key`; the table
// lives in the parameter block, so switching many clients' items in one launch needs no upload.
template <bool CLIENT_KEYS>
__global__ void __launch_bounds__(128) ks_mac_kernel(const u64 *__restrict__ dig, const u64 *__restrict__ key,
                                                    u64 *__restrict__ prod, const __grid_constant__ KsMacConsts c, int n,
                                                    const __grid_constant__ KsKeyTable keys) {
    const int l = c.l, K = c.K;
    const int r = blockIdx.y;
    const int64_t item = blockIdx.z;
    const int coeff = (blockIdx.x * 128 + threadIdx.x) * 2;
    if (coeff >= n) return;
    const int key_row = (r == l) ? K - 1 : r;  // Bfv+Keys.swift:153
    const u64 p = c.p[r], ninv = c.ninv[r];
    u128 a00 = 0, a01 = 0, a10 = 0, a11 = 0;
    const u64 *d = dig + ((item * (l + 1) + r) * l) * n + coeff;
    if (CLIENT_KEYS) key = keys.key[(keys.item0 + item) / keys.items_per_client];
    const u64 *kj = key + (int64_t)key_row * n + coeff;
    for (int j = 0; j < l; ++j) {
        const ulonglong2 dv = *reinterpret_cast<const ulonglong2 *>(d + (int64_t)j * n);
        const ulonglong2 k0 = __ldg(reinterpret_cast<const ulonglong2 *>(kj + (int64_t)j * 2 * K * n));
        const ulonglong2 k1 = __ldg(reinterpret_cast<const ulonglong2 *>(kj + ((int64_t)j * 2 + 1) * K * n));
        mac128(a00, dv.x, k0.x);
        mac128(a01, dv.y, k0.y);
        mac128(a10, dv.x, k1.x);
        mac128(a11, dv.y, k1.y);
    }
    u64 *o = prod + ((item * 2) * (l + 1) + r) * n + coeff;
    *reinterpret_cast<ulonglong2 *>(o) = make_ulonglong2(ks_reduce(a00, p, ninv), ks_reduce(a01, p, ninv));
    *reinterpret_cast<ulonglong2 *>(o + (int64_t)(l + 1) * n) = make_ulonglong2(ks_reduce(a10, p, ninv), ks_reduce(a11, p, ninv));
}

// divide-and-round by the last modulus of `in` (rows c.l), optionally adding `base`, write c.l - 1 rows
__device__ __forceinline__ void divround_column(const u64 *__restrict__ in, const u64 *__restrict__ base,
                                                u64 *__restrict__ out, const DivRoundConsts &c, int64_t n) {
    const int kept = c.l - 1;
    const u64 last = add_mod(in[(int64_t)kept * n], c.half, c.last);  // PolyRq.swift:376-379
    for (int i = 0; i < kept; ++i) {
        const u64 m = c.m[i];
        const u64 tmp = barrett64(last, m, c.mu1[i]);
        u64 v = sub_mod(add_mod(in[(int64_t)i * n], c.half_mod[i], m), tmp, m);
        v = shoup_mul(v, c.inv_w[i], c.inv_wp[i], m);
        if (base) v = add_mod(v, base[(int64_t)i * n], m);
        out[(int64_t)i * n] = v;
    }
}

__global__ void __launch_bounds__(256) ks_finish_kernel(const u64 *__restrict__ prod, const u64 *__restrict__ base,
                                                       int64_t base_item_stride, int base_mask, u64 *__restrict__ out,
                                                       const __grid_constant__ DivRoundConsts c, int64_t n) {
    const int comp = blockIdx.y;
    const int64_t item = blockIdx.z;
    const int64_t coeff = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (coeff >= n) return;
    const int l = c.l - 1;
    const u64 *in = prod + ((item * 2 + comp) * c.l) * n + coeff;
    const u64 *b = (base && ((base_mask >> comp) & 1)) ? base + item * base_item_stride + (int64_t)comp * l * n + coeff : nullptr;
    u64 *o = out + ((item * 2 + comp) * l) * n + coeff;
    divround_column(in, b, o, c, n);
}

__global__ void __launch_bounds__(256) mod_switch_kernel(const u64 *__restrict__ in, u64 *__restrict__ out,
                                                        const __grid_constant__ DivRoundConsts c, int64_t n,
                                                        int64_t total) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int64_t poly = idx / n, coeff = idx - poly * n;
    divround_column(in + poly * c.l * n + coeff, nullptr, out + poly * (c.l - 1) * n + coeff, c, n);
}

cudaError_t launch_ks_mac(const Context &ctx, const u64 *dig, const u64 *key, int l, u64 *prod, int64_t items,
                          cudaStream_t stream, const KsKeyTable *keys) {
    if (items == 0) return cudaSuccess;
    if (ctx.n < 2) return cudaErrorInvalidValue;
    const NttRowMap map = ctx.map_ks(l);
    KsMacConsts c;
    c.l = l;
    c.K = ctx.L + 1;
    for (int r = 0; r <= l; ++r) {
        c.p[r] = ctx.slots[map.slot[r]].dev.p;
        c.ninv[r] = ctx.slots[map.slot[r]].dev.ninv;
    }
    if (keys && keys->items_per_client < 1) return cudaErrorInvalidValue;
    KsKeyTable table = keys ? *keys : KsKeyTable{};
    const unsigned gx = (unsigned)((ctx.n / 2 + 127) / 128);
    return for_each_part(items, [&](int64_t done, int64_t chunk) {
        dim3 grid(gx ? gx : 1, (unsigned)(l + 1), (unsigned)chunk);
        const u64 *d = dig + done * (l + 1) * l * ctx.n;
        u64 *o = prod + done * 2 * (l + 1) * ctx.n;
        if (!keys) return launch(ks_mac_kernel<false>, grid, 128, 0, stream, d, key, o, c, (int)ctx.n, table);
        table.item0 = keys->item0 + done;
        return launch(ks_mac_kernel<true>, grid, 128, 0, stream, d, nullptr, o, c, (int)ctx.n, table);
    });
}

cudaError_t launch_ks_finish(const Context &ctx, const u64 *prod, const u64 *base, int64_t base_item_stride, int base_mask,
                             int l, u64 *out, int64_t items, cudaStream_t stream) {
    if (items == 0) return cudaSuccess;
    const int threads = coeff_threads(ctx.n);
    const DivRoundConsts &c = ctx.ks_divround[l];
    return for_each_part(items, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((ctx.n + threads - 1) / threads), 2, (unsigned)chunk);
        return launch(ks_finish_kernel, grid, threads, 0, stream, prod + done * 2 * (l + 1) * ctx.n,
                      base ? base + done * base_item_stride : nullptr, base_item_stride, base_mask, out + done * 2 * l * ctx.n,
                      c, ctx.n);
    });
}

cudaError_t launch_mod_switch(const Context &ctx, const u64 *in, int l, u64 *out, int64_t polys, cudaStream_t stream) {
    const int64_t total = polys * ctx.n;
    if (total == 0) return cudaSuccess;
    if (l < 2 || l > ctx.L) return cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    return launch(mod_switch_kernel, blocks, 256, 0, stream, in, out, ctx.ms_divround[l], ctx.n, total);
}

}  // namespace hecuda
