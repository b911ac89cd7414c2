// wire_codec.hpp -- what the server calls that answer requests on the wire share (pir.cu, pnns.cu): stream-ordered
// temporaries, the drain of a stream on every return path, and the codec of seeded queries in / packed replies out.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "capi_internal.hpp"

namespace hecuda {
namespace api {

struct StreamBuffers {  // stream-ordered temporaries, freed (stream-ordered) on scope exit
    cudaStream_t s;
    std::vector<void *> ptrs;
    explicit StreamBuffers(cudaStream_t stream) : s(stream) {}
    ~StreamBuffers() {
        for (void *p : ptrs) cudaFreeAsync(p, s);
    }
    cudaError_t alloc(u64 **out, size_t words) { return alloc_bytes((void **)out, std::max<size_t>(words, 1) * sizeof(u64)); }
    cudaError_t alloc_bytes(void **out, size_t bytes) {
        cudaError_t e = cudaMallocAsync(out, std::max<size_t>(bytes, 8), s);
        if (e == cudaSuccess) ptrs.push_back(*out);
        return e;
    }
};

struct DrainOnExit {  // every return path after the caller's buffers are in flight on `s` waits for the stream
    cudaStream_t s;
    ~DrainOnExit() { wait_stream(s); }
};

// Query ciphertexts arrive as SerializedCiphertext.seeded (SerializedCiphertext.swift:41-49: poly0 over all L rows,
// skipLSBs 0, plus the seed; expand_seeded_device turns them into Coeff ciphertexts).  Replies leave as
// .full(polys:skipLSBs:) with Bfv.skipLSBsForDecryption (Bfv+Decrypt.swift:51-110): single-modulus ciphertexts whose
// poly 0 and poly 1 are packed with different numbers of dropped low bits.
struct WireCodec {
    CodecConsts in, out[2];
    int skip[2] = {0, 0};
    size_t query_bytes = 0, bytes[2] = {0, 0};  // one serialized query poly0; one packed reply poly 0 / poly 1
    u64 *polys = nullptr;                        // 2 x replies x N: poly p of every reply, contiguous
    unsigned char *packed[2] = {nullptr, nullptr}, *reply = nullptr;  // replies x bytes[p]; replies x reply_bytes()
    size_t reply_bytes() const { return bytes[0] + bytes[1]; }
    int32_t setup(const Context &c, int skip0, int skip1) {
        std::string err;
        if (!codec_consts(c, c.map_q(c.L), 0, in, err) || !codec_consts(c, c.map_q(1), skip0, out[0], err) ||
            !codec_consts(c, c.map_q(1), skip1, out[1], err))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
        skip[0] = skip0, skip[1] = skip1;
        query_bytes = (size_t)serialized_poly_bytes(in);
        for (int p = 0; p < 2; ++p) bytes[p] = (size_t)serialized_poly_bytes(out[p]);
        return HECUDA_OK;
    }
    cudaError_t alloc(StreamBuffers &tmp, const Context &c, int64_t replies) {  // buffers for up to `replies` replies
        cudaError_t e = tmp.alloc(&polys, (size_t)2 * c.n * replies);
        for (int p = 0; p < 2 && e == cudaSuccess; ++p)
            e = tmp.alloc_bytes((void **)&packed[p], ((bytes[p] + 7) & ~(size_t)7) * replies + 8);
        if (e == cudaSuccess) e = tmp.alloc_bytes((void **)&reply, reply_bytes() * replies);
        return e;
    }
    // resp: replies x 2 x 1 x N (Coeff) -> reply: replies x (bytes[0] + bytes[1])
    int32_t pack(const Context &c, const u64 *resp, int64_t replies, cudaStream_t s) {
        const size_t pw = (size_t)c.n * sizeof(u64);
        for (int p = 0; p < 2; ++p) {
            CK(cudaMemcpy2DAsync(polys + (size_t)p * c.n * replies, pw, resp + (size_t)p * c.n, 2 * pw, pw, (size_t)replies,
                                 cudaMemcpyDeviceToDevice, s));
            cudaError_t e = launch_poly_serialize(c, out[p], skip[p], polys + (size_t)p * c.n * replies, packed[p], replies, s);
            if (e != cudaSuccess) return cuda_fail(e, "serialize response");
            CK(cudaMemcpy2DAsync(reply + (p ? bytes[0] : 0), reply_bytes(), packed[p], bytes[p], bytes[p], (size_t)replies,
                                 cudaMemcpyDeviceToDevice, s));
        }
        return HECUDA_OK;
    }
};

}  // namespace api
}  // namespace hecuda
