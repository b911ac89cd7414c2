// ntt.cu -- dispatch between the NTT implementations.
//   register-tiled kernels (ntt_fast.cu) for N = 2^10 .. 2^14, generic radix-2 shared-memory kernel
//   (ntt_simple.cu) otherwise; HECUDA_NTT_IMPL=simple forces the latter (A/B testing).
#include <cstdlib>
#include <cstring>

#include "kernels.cuh"

namespace hecuda {

static bool use_fast(const Context &ctx) {
    static const bool forced_simple = [] {
        const char *e = std::getenv("HECUDA_NTT_IMPL");
        return e && !std::strcmp(e, "simple");
    }();
    return !forced_simple && ntt_fast_supported(ctx);
}

cudaError_t launch_ntt_forward(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               cudaStream_t stream) {
    if (use_fast(ctx)) return launch_ntt_forward_fast(ctx, map, in, out, rows, stream);
    return launch_ntt_forward_simple(ctx, map, in, out, rows, stream);
}

cudaError_t launch_ntt_inverse(const Context &ctx, const NttRowMap &map, const u64 *in, u64 *out, int64_t rows,
                               int scale_mode, cudaStream_t stream) {
    if (use_fast(ctx)) return launch_ntt_inverse_fast(ctx, map, in, out, rows, scale_mode, stream);
    return launch_ntt_inverse_simple(ctx, map, in, out, rows, scale_mode, stream);
}

bool ntt_forward_tensor_supported(const Context &ctx) { return use_fast(ctx) && ctx.logn == 13; }

}  // namespace hecuda
