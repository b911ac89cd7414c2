// cuckoo.hpp -- CuckooTable placement (KeywordPir/CuckooTable.swift), host C++.
//
// The insertion loop is sequential by design: the table it builds depends on the order of the generator's draws, and
// that order is what the reference's tests pin.  Everything around it is data-parallel and runs on the device
// (keyword_pir.cu): the caller supplies the candidate indices of every entry for a given bucketsPerTable through a
// callback, computed there by one kernel launch per bucket count the placement reaches (in tests/emu by host SHA-256).
//
// Entries are ids into the caller's rows.  A bucket holds entry ids in slot order and its serialized size, which is
// kept up to date on every change instead of being recomputed from the values.
//
// One deliberate divergence from the reference: when no candidate bucket has a swap index, CuckooTable.insertLoop
// (CuckooTable.swift:455-457) expands the table and returns without inserting the pair in hand -- a new row or one just
// evicted, so that row is silently lost.  Here the pair is inserted again after the expansion, as the branch at
// :402-406 does.  Tables are identical to the reference's whenever that branch is not taken.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace hecuda {
namespace cuckoo {

struct Config {
    int hash_function_count;
    int64_t max_eviction_count;
    int64_t max_serialized_bucket_size;
    int slot_count;
    bool multiple_tables;
    int64_t fixed_bucket_count;  // 0: .allowExpansion
    double expansion_factor, target_load_factor;
    int table_count() const { return multiple_tables ? hash_function_count : 1; }
};

// HashBucket.serializedSize
inline int64_t bucket_header_size() { return 1; }
inline int64_t slot_size(int64_t value_length) { return 10 + value_length; }

// CuckooTableConfig.validate (CuckooTable.swift:138-156); "" when valid.  Two cases the reference accepts but cannot
// build a table with are refused as well: a target load factor <= 0 (Int(ceil(x / 0)) traps) and, with expansion,
// maxEvictionCount < 1 (insert and expand call each other without end).
inline std::string validate(const Config &c) {
    bool ok = c.hash_function_count > 0 && c.max_serialized_bucket_size >= bucket_header_size() + slot_size(0) &&
              c.slot_count > 0 && c.slot_count <= 255 && c.max_eviction_count >= 0;
    if (c.fixed_bucket_count == 0)
        ok = ok && c.expansion_factor > 1.0 && c.target_load_factor < 1.0 && c.target_load_factor > 0.0 &&
             c.max_eviction_count >= 1;
    else
        ok = ok && c.max_serialized_bucket_size > 0 && c.fixed_bucket_count > 0;
    return ok ? "" : "invalidCuckooConfig";
}

inline int64_t next_multiple(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// Random-number generators; `bounded` is Swift's RandomNumberGenerator.next(upperBound:), which
// Collection.randomElement(using:) reaches through Int.random(in: 0..<n).
struct Generator {
    enum Kind { kCounter = 0, kSplitMix64 = 1 };
    int kind;
    uint64_t state;
    uint64_t next() {
        if (kind == kCounter) return state++;  // _TestUtilities TestRng: the counter, then += 1
        uint64_t z = (state += 0x9e3779b97f4a7c15ull);
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        return z ^ (z >> 31);
    }
    uint64_t bounded(uint64_t n) {
        unsigned __int128 m = (unsigned __int128)next() * n;
        if ((uint64_t)m < n) {
            const uint64_t t = (0 - n) % n;
            while ((uint64_t)m < t) m = (unsigned __int128)next() * n;
        }
        return (uint64_t)(m >> 64);
    }
};

struct Failure {
    std::string message;
};

struct Bucket {
    std::vector<int64_t> slots;  // entry ids, in slot order
    int64_t size = 1;            // serialized size
};

// Rows: count keyword/value pairs.  candidates(bucketsPerTable) -> count x h candidate indices (HashKeyword.hashIndices
// for every entry), valid until the next call; it is called again only when bucketsPerTable changes.
template <class Candidates>
class Table {
  public:
    Table(const Config &config, int64_t count, const unsigned char *keywords, const uint64_t *keyword_offsets,
          const uint64_t *hashes, const uint64_t *value_offsets, Generator rng, Candidates candidates)
        : config_(config), count_(count), keywords_(keywords), keyword_offsets_(keyword_offsets), hashes_(hashes),
          value_offsets_(value_offsets), rng_(rng), candidates_(std::move(candidates)) {}

    // CuckooTable.init (CuckooTable.swift:328-357): rows inserted in order
    void build() {
        int64_t target;
        if (config_.fixed_bucket_count == 0) {
            int64_t total = bucket_header_size();
            for (int64_t e = 0; e < count_; ++e) total += slot_size(value_length(e));
            const int64_t min_buckets = (total + config_.max_serialized_bucket_size - 1) / config_.max_serialized_bucket_size;
            target = next_multiple((int64_t)std::ceil((double)min_buckets / config_.target_load_factor), config_.table_count());
        } else {
            target = next_multiple(config_.fixed_bucket_count, config_.table_count());
        }
        buckets_.assign((size_t)target, Bucket());
        for (int64_t e = 0; e < count_; ++e) insert(e);
    }

    const std::vector<Bucket> &buckets() const { return buckets_; }
    int64_t buckets_per_table() const { return (int64_t)buckets_.size() / config_.table_count(); }

  private:
    int64_t value_length(int64_t e) const { return (int64_t)(value_offsets_[e + 1] - value_offsets_[e]); }
    bool same_keyword(int64_t a, int64_t b) const {
        if (hashes_[a] != hashes_[b]) return false;
        const uint64_t la = keyword_offsets_[a + 1] - keyword_offsets_[a], lb = keyword_offsets_[b + 1] - keyword_offsets_[b];
        return la == lb && std::memcmp(keywords_ + keyword_offsets_[a], keywords_ + keyword_offsets_[b], la) == 0;
    }
    int64_t index(int table, int64_t i) const {  // CuckooTable.index(tableIndex:index:), :461-463
        return config_.table_count() == 1 ? i : table * buckets_per_table() + i;
    }
    const int64_t *candidates_of(int64_t e) {
        const int64_t per_table = buckets_per_table();
        if (per_table != cached_per_table_) {
            cached_ = candidates_(per_table);
            cached_per_table_ = per_table;
        }
        return cached_ + e * config_.hash_function_count;
    }

    // CuckooTable.insert (:386-398)
    void insert(int64_t e) {
        if (bucket_header_size() + slot_size(value_length(e)) > config_.max_serialized_bucket_size)
            throw Failure{"failedToConstructCuckooTable: a " + std::to_string(value_length(e)) +
                          "-byte value makes a hash bucket larger than maxSerializedBucketSize"};
        insert_loop(e, config_.max_eviction_count);
    }

    // CuckooTable.insertLoop (:400-458), its tail recursion as a loop
    void insert_loop(int64_t e, int64_t remaining) {
        const int h = config_.hash_function_count;
        for (;;) {
            if (remaining == 0) {
                if (config_.fixed_bucket_count != 0)
                    throw Failure{"failedToConstructCuckooTable: unable to insert into a table with " +
                                  std::to_string(entry_count()) +
                                  " entries; consider allowExpansion or a larger bucketCount"};
                expand();
                insert(e);
                // the reference falls through to the checks below, which find the pair just inserted
            }
            const int64_t *cand = candidates_of(e);
            for (int t = 0; t < h; ++t)  // the keyword is already present
                for (int64_t other : buckets_[(size_t)index(t, cand[t])].slots)
                    if (same_keyword(other, e)) return;
            const int64_t grow = slot_size(value_length(e));
            for (int t = 0; t < h; ++t) {  // first fit: CuckooBucket.canInsert (:202-205)
                Bucket &b = buckets_[(size_t)index(t, cand[t])];
                if ((int64_t)b.slots.size() < config_.slot_count && b.size + grow <= config_.max_serialized_bucket_size) {
                    b.slots.push_back(e);
                    b.size += grow;
                    return;
                }
            }
            swaps_.clear();  // CuckooBucket.swapIndices (:209-217) of every candidate, in table order
            for (int t = 0; t < h; ++t) {
                const int64_t at = index(t, cand[t]);
                const Bucket &b = buckets_[(size_t)at];
                for (size_t s = 0; s < b.slots.size(); ++s)
                    if (b.size - slot_size(value_length(b.slots[s])) + grow <= config_.max_serialized_bucket_size)
                        swaps_.emplace_back(at, (int64_t)s);
            }
            if (swaps_.empty()) {
                expand();
                insert(e);  // the divergence: the reference drops the pair here
                return;
            }
            const std::pair<int64_t, int64_t> pick = swaps_[(size_t)rng_.bounded(swaps_.size())];
            Bucket &b = buckets_[(size_t)pick.first];
            const int64_t evicted = b.slots[(size_t)pick.second];
            b.slots[(size_t)pick.second] = e;
            b.size += grow - slot_size(value_length(evicted));
            e = evicted;
            --remaining;
        }
    }

    // CuckooTable.expand (:466-490): the old buckets re-inserted in order, nested expansions as they happen
    void expand() {
        if (config_.fixed_bucket_count != 0)
            throw Failure{"failedToConstructCuckooTable: needed to expand a table that does not allow expansion"};
        std::vector<Bucket> old;
        old.swap(buckets_);
        const int64_t count = next_multiple((int64_t)std::ceil((double)old.size() * config_.expansion_factor),
                                            config_.table_count());
        buckets_.assign((size_t)count, Bucket());
        for (const Bucket &b : old)
            for (int64_t e : b.slots) insert(e);
    }

    int64_t entry_count() const {
        int64_t n = 0;
        for (const Bucket &b : buckets_) n += (int64_t)b.slots.size();
        return n;
    }

    Config config_;
    int64_t count_;
    const unsigned char *keywords_;
    const uint64_t *keyword_offsets_, *hashes_, *value_offsets_;
    Generator rng_;
    Candidates candidates_;
    std::vector<Bucket> buckets_;
    std::vector<std::pair<int64_t, int64_t>> swaps_;
    const int64_t *cached_ = nullptr;
    int64_t cached_per_table_ = -1;
};

}  // namespace cuckoo
}  // namespace hecuda
