// proto_respond.hpp -- what every server that answers the reference's protobuf messages on the device shares (PIR,
// pir.cu; PNNS, pnns.cu): the offset tables that let the seeded expansion read a group's query ciphertexts in place
// from its uploaded messages, and the framing of the replies from one client's template.
//
// A reply message is its framing (every byte that is not a reply poly) plus the polys, which the packing kernels
// write straight into their slots.  The framing is the same for every client of a call, so the host builds it once as
// runs (offset in the message, bytes) and one launch per group copies every run into every client's message.
#pragma once
#include <algorithm>
#include <cuda_runtime.h>
#include <utility>
#include <vector>

#include "he_proto.hpp"

namespace hecuda {
namespace api {

// One client's framing: run i puts bytes[from_i, from_i + length_i) at offset at_i of the client's `size`-byte message.
// `table` holds (at, from, length) triples; runs longer than kFrameRunBytes are split so that no block copies more.
struct FrameRuns {
    static constexpr long long kFrameRunBytes = 4096;
    std::vector<long long> table;
    proto::Bytes bytes;
    long long size = 0;
    void put(long long at, const unsigned char *b, long long length) {
        for (long long done = 0; done < length; done += kFrameRunBytes) {
            table.push_back(at + done);
            table.push_back((long long)bytes.size() + done);
            table.push_back(std::min(kFrameRunBytes, length - done));
        }
        bytes.insert(bytes.end(), b, b + length);
    }
    void put(long long at, const proto::Bytes &b) { put(at, b.data(), (long long)b.size()); }
    long long runs() const { return (long long)table.size() / 3; }
};

// Every run of `f` (uploaded: d_table, d_bytes) into each of `clients` messages of f.size bytes at d_out: one launch
cudaError_t launch_frame_runs(unsigned char *d_out, int clients, long long size, const long long *d_table, long long runs,
                              const unsigned char *d_bytes, cudaStream_t s);

// One group's query ciphertexts read in place from its messages (uploaded back to back at msg_at[j]): the offset tables
// of the seeded expansion (tag: poly0, frame 0, a .full ciphertext's entry equal to the next one's so that it expands
// to zero rows; seed: its seed, or `pad` for a .full one), then per distinct skip value the .full polys' offsets and
// their slots in the group's batch x 2 x L x N query buffer.  cts[j]: client j's ciphertexts, offsets into its message.
struct GroupTables {
    std::vector<long long> tag, seed;
    std::vector<std::pair<int, std::vector<long long>>> full;  // skip -> offsets, then slots (half and half)
};
inline GroupTables group_tables(const std::vector<const std::vector<heproto::Ciphertext> *> &cts_of,
                                const std::vector<long long> &msg_at, long long pad) {
    GroupTables t;
    const size_t cts = cts_of[0]->size(), batch = cts * cts_of.size();
    t.tag.assign(batch + 1, 0);
    t.seed.assign(batch, pad);
    t.tag[batch] = pad + 1;  // past every poly0
    std::vector<std::pair<int, std::pair<long long, long long>>> polys;  // (skip, (offset, slot))
    for (size_t b = batch; b-- > 0;) {
        const heproto::Ciphertext &ct = (*cts_of[b / cts])[b % cts];
        const long long base = msg_at[b / cts];
        t.tag[b] = ct.full ? t.tag[b + 1] : base + ct.poly[0];
        if (!ct.full) {
            t.seed[b] = base + ct.seed;
            continue;
        }
        for (int p = 1; p >= 0; --p) polys.push_back({ct.skip[p], {base + ct.poly[p], (long long)(2 * b + p)}});
    }
    std::reverse(polys.begin(), polys.end());  // message order: the offsets increase
    for (const auto &q : polys) {
        auto it = std::find_if(t.full.begin(), t.full.end(), [&](const auto &f) { return f.first == q.first; });
        if (it == t.full.end()) it = t.full.insert(t.full.end(), {q.first, {}});
        it->second.push_back(q.second.first);
    }
    for (auto &f : t.full) {  // offsets (plus a sentinel past the last), then the slots
        f.second.push_back(f.second.back() + 1);
        for (const auto &q : polys)
            if (q.first == f.first) f.second.push_back(q.second.second);
    }
    return t;
}

}  // namespace api
}  // namespace hecuda
