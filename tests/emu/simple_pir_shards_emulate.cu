// Host replay of sharded SimplePIR's index maps (swift-homomorphic-encryption_b200/csrc/simple_pir.cuh): the chunk
// locations' inversion and the row -> piece map the shard pack kernel reads, and the grouped response kernel's plan
// and work-item decode.
//
//   rows              stdin: entry_count shard_count chunk_size, the entry sizes, their bytes, then 2 x chunks
//                     locations (shard, index) -> "refused", or "ok" then every shard's rows as hex, one per line
//   items sms max_shards min_split_tiles
//                     stdin: shard_count, then m col_tiles q per shard -> one line per work item of every launch:
//                     launch shard row_cta pair k_begin k_end
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../swift-homomorphic-encryption_b200/csrc/simple_pir.cuh"

using namespace hecuda;

int main(int argc, char **argv) {
    if (argc >= 2 && !strcmp(argv[1], "rows")) {
        long long entries, chunk_size;
        int shards;
        if (scanf("%lld %d %lld", &entries, &shards, &chunk_size) != 3) return 2;
        std::vector<uint64_t> offsets(entries + 1, 0);
        for (long long e = 0; e < entries; ++e) {
            long long size;
            scanf("%lld", &size);
            offsets[e + 1] = offsets[e] + size;
        }
        std::vector<unsigned char> values(offsets[entries] + 1);
        for (uint64_t i = 0; i < offsets[entries]; ++i) {
            unsigned v;
            scanf("%u", &v);
            values[i] = (unsigned char)v;
        }
        long long chunks = 0;
        for (long long e = 0; e < entries; ++e) chunks += (long long)((offsets[e + 1] - offsets[e] + chunk_size - 1) / chunk_size);
        std::vector<int64_t> locations(2 * chunks);
        for (auto &v : locations) scanf("%lld", (long long *)&v);
        std::vector<long long> row_begin(shards + 1), row_source(2 * chunks);
        if (!spir::shard_rows(offsets.data(), entries, chunk_size, locations.data(), shards, row_begin.data(), row_source.data())) {
            printf("refused\n");
            return 0;
        }
        printf("ok\n");
        procdb::PirShape s{};
        s.entries = values.data();
        s.offsets = offsets.data();
        s.entry_count = entries;
        s.entry_size = chunk_size;
        s.encoded = chunk_size;
        for (int sh = 0; sh < shards; ++sh)
            for (long long r = row_begin[sh]; r < row_begin[sh + 1]; ++r) {
                const procdb::PirPiece p = spir::shard_piece(s, row_source[2 * r], row_source[2 * r + 1], chunk_size);
                printf("%d ", sh);
                for (long long j = 0; j < chunk_size; ++j) printf("%02x", j < p.length ? procdb::pir_piece_byte(s, p, j) : 0u);
                printf("\n");
            }
        return 0;
    }
    if (argc >= 5 && !strcmp(argv[1], "items")) {
        const int sms = atoi(argv[2]), max_shards = atoi(argv[3]), min_split = atoi(argv[4]);
        int count;
        if (scanf("%d", &count) != 1) return 2;
        std::vector<long long> m(count), col_tiles(count), q(count), items(count);
        std::vector<spir::ItemShape> shape(count);
        long long ctas = 0;
        for (int s = 0; s < count; ++s) {
            scanf("%lld %lld %lld", &m[s], &col_tiles[s], &q[s]);
            ctas += spir::base_ctas(m[s], q[s]);
        }
        for (int s = 0; s < count; ++s) {
            shape[s] = spir::item_shape(m[s], col_tiles[s], q[s], ctas, sms, min_split);
            items[s] = spir::item_count(shape[s]);
        }
        int launch = 0;
        for (int first = 0, end = 0; first < count; first = end, ++launch) {
            end = spir::group_end(items.data(), first, count, max_shards, INT_MAX);
            std::vector<long long> begin;
            long long total = 0;
            for (int s = first; s < end; ++s) {
                begin.push_back(total);
                total += items[s];
            }
            for (long long item = 0; item < total; ++item) {
                const int local = spir::item_shard(begin.data(), end - first, item);
                const int s = first + local;
                long long row_cta, pair, kb, ke;
                spir::decode_item(shape[s], col_tiles[s], item - begin[local], row_cta, pair, kb, ke);
                printf("%d %d %lld %lld %lld %lld\n", launch, s, row_cta, pair, kb, ke);
            }
        }
        return 0;
    }
    fprintf(stderr, "usage: rows | items sms max_shards min_split_tiles\n");
    return 2;
}
