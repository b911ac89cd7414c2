// oprf_host.hpp -- host-side argument checks and buffer helpers shared by the OPRF server (symmetric_pir.cu) and the
// OPRF client (oprf_client.cu).
#pragma once
#include <algorithm>
#include <string>

#include "capi_internal.hpp"

namespace hecuda {
namespace api {
namespace oprf_host {

constexpr long long kMaxInputBytes = 65535;  // I2OSP(len(input), 2)

inline void wipe(void *p, size_t bytes) {  // a host copy of key material
    volatile unsigned char *q = (volatile unsigned char *)p;
    for (size_t i = 0; i < bytes; ++i) q[i] = 0;
}

// offsets[0..count] must not decrease; `longest` gets the longest row
inline int32_t check_rows(const uint64_t *offsets, int64_t count, const char *what, uint64_t &longest) {
    longest = 0;
    for (int64_t i = 0; i < count; ++i) {
        if (offsets[i + 1] < offsets[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, std::string(what) + " offsets must not decrease");
        longest = std::max<uint64_t>(longest, offsets[i + 1] - offsets[i]);
    }
    return HECUDA_OK;
}

inline int32_t check_inputs(const uint8_t *inputs, const uint64_t *offsets, int64_t count, const char *what) {
    if (!inputs || !offsets || count < 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / negative count");
    uint64_t longest = 0;
    const int32_t rc = check_rows(offsets, count, what, longest);
    if (rc) return rc;
    if (longest > (uint64_t)kMaxInputBytes)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, std::string(what) + " longer than 65535 bytes (OPRF inputs carry a 2-byte length)");
    return HECUDA_OK;
}

inline int32_t have_device() {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(HECUDA_ERR_NO_DEVICE, "no CUDA device: libhecuda has no CPU fallback");
    return HECUDA_OK;
}

template <class T>
cudaError_t upload_new(T **dst, const void *src, size_t bytes) {
    cudaError_t e = cudaMalloc(dst, std::max<size_t>(bytes, 1));
    if (e == cudaSuccess && bytes) e = upload(*dst, src, bytes);
    return e;
}

}  // namespace oprf_host
}  // namespace api
}  // namespace hecuda
