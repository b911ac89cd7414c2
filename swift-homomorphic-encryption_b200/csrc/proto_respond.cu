// proto_respond.cu -- the framing launch of the protobuf reply paths (proto_respond.hpp)
#include "capi_internal.hpp"
#include "proto_respond.hpp"

namespace hecuda {
namespace api {

namespace {

// one CTA per (run, client): run blockIdx.x of the template into client blockIdx.y's message
__global__ void __launch_bounds__(128) frame_runs_kernel(unsigned char *__restrict__ out, long long size,
                                                         const long long *__restrict__ table,
                                                         const unsigned char *__restrict__ bytes) {
    const long long *run = table + 3 * (long long)blockIdx.x;
    const long long at = run[0], from = run[1], length = run[2];
    unsigned char *dst = out + (long long)blockIdx.y * size + at;
    for (long long k = threadIdx.x; k < length; k += blockDim.x) dst[k] = bytes[from + k];
}

}  // namespace

cudaError_t launch_frame_runs(unsigned char *d_out, int clients, long long size, const long long *d_table, long long runs,
                              const unsigned char *d_bytes, cudaStream_t s) {
    if (runs == 0 || clients == 0) return cudaSuccess;
    if (runs > 0x7fffffffLL || clients > 65535) return cudaErrorInvalidValue;
    return launch(frame_runs_kernel, dim3((unsigned)runs, (unsigned)clients), 128, 0, s, d_out, size, d_table, d_bytes);
}

}  // namespace api
}  // namespace hecuda
