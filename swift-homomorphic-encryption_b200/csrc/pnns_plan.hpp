// pnns_plan.hpp -- the query plan of PlaintextMatrix.mulTranspose(matrix:) on the host: what extractDenseRow derives
// for every row of a `.denseRow` query, and the single rotations of the packing step.  Only the query's and the
// database's dimensions and the client's Galois elements enter it, so a server that learns the query's shape from a
// message can answer it with nothing else.
//
//   CiphertextMatrix.ciphertextCount / extractDenseRow     CiphertextMatrix.swift:245-352
//   GaloisElement.rotatingColumns / stepsFor / _planMultiStep   PolyRq/Galois.swift:195-319
//   rotateColumnsMultiStep(by:)                            _HomomorphicEncryptionExtras/HeScheme.swift:65-104
//
// hecuda/pnns.py's PlaintextMatrix._rowDescriptors derives the same plan in Python; tests/emu/pnns_proto_emulate.cu
// checks the two agree.
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace hecuda {
namespace pnnsplan {

inline int64_t next_pow2(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

// CiphertextMatrix.ciphertextCount of a .denseRow matrix (rows x columns, columns <= N / 2)
inline int64_t ciphertext_count(int64_t n, int64_t rows, int64_t columns) {
    const int64_t per_ciphertext = 2 * ((n / 2) / next_pow2(columns));
    return (rows + per_ciphertext - 1) / per_ciphertext;
}

// extractDenseRow for row `row` (CiphertextMatrix.swift:254-320): the ciphertext holding it, its 0/1 SIMD mask (the
// first `mask.size()` of N slots; the rest are 0) and its number of rotate-and-add replication steps
struct RowExtraction {
    int32_t ciphertext = 0, rotations = 0;
    std::vector<uint8_t> mask;
};
inline RowExtraction dense_row_extraction(int64_t n, int64_t rows, int64_t columns, int64_t ciphertexts, int64_t row) {
    const int64_t half = n / 2, width = next_pow2(columns), per_ciphertext = 2 * (half / width);
    RowExtraction x;
    x.ciphertext = (int32_t)(row / per_ciphertext);
    const bool last = x.ciphertext == ciphertexts - 1;
    auto slots = [&](int64_t r, int64_t &lo, int64_t &hi) {
        lo = (r % per_ciphertext) * width;
        hi = lo + width;
        if (lo <= half && half < hi) {  // the batch would straddle the two SIMD rows
            lo = half, hi = half + width;
        } else if (hi > half) {  // second SIMD row: skip the first row's padding
            lo += half % width, hi += half % width;
        }
        if (last) hi = (hi + half - 1) / half * half;  // the last ciphertext repeats its rows to the end
    };
    int64_t lo, hi, l2, h2;
    slots(row, lo, hi);
    int64_t after = row + 1;
    while (after < rows && (slots(after, l2, h2), h2 == hi)) ++after;
    int64_t before = std::max<int64_t>(row - 1, 0);
    while (before > 0 && (slots(before, l2, h2), h2 == hi)) --before;
    const int64_t period = next_pow2(width * (after - before));
    x.mask.assign((size_t)lo, 0);
    int64_t copies = 0;
    while ((int64_t)x.mask.size() < hi) {
        x.mask.insert(x.mask.end(), (size_t)width, 1);
        x.mask.insert(x.mask.end(), (size_t)(period - width), 0);
        ++copies;
    }
    if ((int64_t)x.mask.size() > n) x.mask.resize((size_t)n);
    x.rotations = (int32_t)(half / (copies * width) - 1);
    return x;
}

// GaloisElement.rotatingColumns(by:degree:): 0 for a step outside (0, N/2) in magnitude (invalidRotationStep)
inline uint64_t rotating_columns(int64_t step, int64_t n) {
    int64_t positive = step < 0 ? -step : step;
    if (!(0 < positive && positive < n / 2)) return 0;
    if (step > 0) positive = n / 2 - positive;
    uint64_t g = 1, base = 3, mod = 2 * (uint64_t)n;
    for (int64_t e = positive; e; e >>= 1) {
        if (e & 1) g = g * base % mod;
        base = base * base % mod;
    }
    return g;
}

// GaloisElement.stepsFor: the rotation step of every element that is a power of 3 mod 2N (3^k <-> N/2 - k, the first k)
inline std::vector<int64_t> steps_for(const std::set<uint64_t> &elements, int64_t n) {
    std::map<uint64_t, int64_t> found;
    uint64_t g = 1;
    for (int64_t k = 0; k <= n / 2; ++k) {
        if (elements.count(g) && !found.count(g)) found[g] = n / 2 - k;
        g = g * 3 % (2 * (uint64_t)n);
    }
    std::vector<int64_t> steps;
    for (const auto &f : found) steps.push_back(f.second);
    return steps;
}

// GaloisElement._planMultiStep: a greedy decomposition by the steps, or by their complements to N/2, whichever needs
// fewer rotations (the steps' plan on a tie); false when neither decomposes `step`
inline bool plan_multi_step(const std::vector<int64_t> &supported, int64_t step, int64_t n, std::map<int64_t, int64_t> &plan) {
    plan.clear();
    if (std::find(supported.begin(), supported.end(), step) != supported.end()) {
        plan[step] = 1;
        return true;
    }
    std::vector<int64_t> down(supported);
    std::sort(down.rbegin(), down.rend());
    auto greedy = [&](bool forward, std::map<int64_t, int64_t> &out) {
        int64_t left = forward ? step : n / 2 - step;
        out.clear();
        for (size_t i = 0; i < down.size(); ++i) {
            const int64_t s = forward ? down[i] : down[down.size() - 1 - i], w = forward ? s : n / 2 - s;
            if (w <= 0) continue;
            if (left / w) out[s] += left / w;
            left %= w;
        }
        return left == 0;
    };
    std::map<int64_t, int64_t> fwd, bwd;
    const bool has_f = greedy(true, fwd), has_b = greedy(false, bwd);
    if (!has_f && !has_b) return false;
    if (!has_b || (has_f && [&] {
            int64_t a = 0, b = 0;
            for (const auto &p : fwd) a += p.second;
            for (const auto &p : bwd) b += p.second;
            return a <= b;
        }()))
        plan = fwd;
    else
        plan = bwd;
    return true;
}

// The single rotations of rotateColumnsMultiStep(by: step), larger steps first; false: invalidRotationStep
inline bool rotation_sequence(const std::set<uint64_t> &elements, int64_t step, int64_t n, std::vector<int32_t> &out) {
    out.clear();
    if (step == 0) return true;
    const uint64_t direct = rotating_columns(step, n);
    if (direct == 0) return false;
    if (elements.count(direct)) {
        out.push_back((int32_t)step);
        return true;
    }
    const int64_t want = step < 0 ? step + n / 2 : step;
    if ((want < 0 ? -want : want) >= n) return false;
    std::map<int64_t, int64_t> plan;
    if (!plan_multi_step(steps_for(elements, n), want, n, plan)) return false;
    for (auto it = plan.rbegin(); it != plan.rend(); ++it)
        for (int64_t k = 0; k < it->second; ++k) out.push_back((int32_t)it->first);
    return true;
}

// Everything mulTranspose(matrix:) needs for a query of `rows` x `columns` against a database of `db_rows` rows:
// the arguments hecuda_pnns_mul_transpose_matrix takes, with the masks as 0/1 SIMD values (rows x N) still to encode
struct QueryPlan {
    int32_t rows = 0, column_step = 0;
    int64_t ciphertexts = 0;
    std::vector<int32_t> index, rotate, pack;
    std::vector<uint64_t> mask_values;  // rows x N; empty for a single row
};
inline bool plan_query(int64_t n, int64_t rows, int64_t columns, int64_t db_rows, const std::set<uint64_t> &elements,
                       QueryPlan &p, std::string &err) {
    p = QueryPlan{};
    p.rows = (int32_t)rows;
    p.ciphertexts = ciphertext_count(n, rows, columns);
    p.column_step = (int32_t)next_pow2(columns);
    p.index.assign((size_t)rows, 0);
    p.rotate.assign((size_t)rows, 0);
    if (rows > 1) {
        p.mask_values.assign((size_t)(rows * n), 0);
        for (int64_t r = 0; r < rows; ++r) {
            const RowExtraction x = dense_row_extraction(n, rows, columns, p.ciphertexts, r);
            p.index[(size_t)r] = x.ciphertext, p.rotate[(size_t)r] = x.rotations;
            std::copy(x.mask.begin(), x.mask.end(), p.mask_values.begin() + r * n);
        }
    }
    if ((n / 2) / db_rows > 1 && rows > 1 && !rotation_sequence(elements, db_rows, n, p.pack)) {
        err = "invalidRotationStep(step: " + std::to_string(db_rows) + ", degree: " + std::to_string(n) + ")";
        return false;
    }
    return true;
}

}  // namespace pnnsplan
}  // namespace hecuda
