// pnns.cu -- PNNS server: encrypted-vector x plaintext-matrix product on one device (SURVEY.md 8f rank 3).
//
//   PlaintextMatrix.mulTranspose(vector:using:)    PrivateNearestNeighborSearch/MatrixMultiplication.swift:131-226
//   BabyStepGiantStep                              MatrixMultiplication.swift:26-62
//   rotateColumnsAndSum                            _HomomorphicEncryptionExtras/HeScheme.swift:113-134
//   Server.computeResponse post-processing         PrivateNearestNeighborSearch/Server.swift:61-88
//
// The matrix stays in HBM in Eval format, re-ordered once so that every (result ciphertext, giant step) pair owns
// `babyStep` consecutive plaintexts (absent ones flagged), which makes step 2 of the algorithm a single launch of the
// streaming ct x pt inner-product kernel per query vector.  Query vectors that share an evaluation key are batched
// through the rotation chains (babyStep - 1 rotations by -1, giantStep - 1 rotations by -babyStep).
//
// Many clients, each with its own evaluation key, are answered in groups of up to HECUDA_PNNS_CLIENT_GROUP: every
// buffer is client-major, each rotation is one key-switching pass over the whole group with a per-client key table,
// and the matrix streams once per group (the many-clients scan).  A group of one issues the single-client launches.
#include <algorithm>
#include <set>

#include "capi_internal.hpp"
#include "wire_codec.hpp"

using namespace hecuda;
using namespace hecuda::api;

struct hecuda_pnns_matrix {
    const hecuda_context *owner = nullptr;
    u64 *d_plain = nullptr;              // [result][giant][baby] x L x N, Eval
    unsigned char *d_present = nullptr;  // [result][giant][baby]
    int64_t row_count = 0, column_count = 0, result_count = 0;
    int baby = 0, giant = 0, dimension = 0;
};

namespace {

static_assert(HECUDA_PNNS_CLIENT_GROUP == kKeyTableSize, "one key-table entry per client of a group");

// Where the items of an accumulate live: they form clients of `per_client` items each, and item k of client j is the
// ciphertext at acc + j * acc_client + k * (2 x rows x N) and at src + j * src_client + k * src_stride (all in words).
struct AccLayout {
    long long per_client, src_stride, src_client, acc_client;
};

// acc[item] (+)= src[item]   over ciphertexts of 2 x rows x N
// modes (optional, per item): 0 = leave acc alone, 1 = copy, 2 = add; without modes every item uses `add`
__global__ void __launch_bounds__(256) accumulate_kernel(u64 *__restrict__ acc, const u64 *__restrict__ src,
                                                        const __grid_constant__ AccLayout lay, long long item0,
                                                        const __grid_constant__ RowModuli c, int n, int add,
                                                        const signed char *__restrict__ modes) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const long long item = item0 + blockIdx.z;
    if (modes) {
        const int mode = modes[item];
        if (mode == 0) return;
        add = mode == 2;
    }
    const long long client = item / lay.per_client, k = item - client * lay.per_client;
    const int pr = blockIdx.y;
    const int64_t ct_words = (int64_t)2 * c.rows * n;
    const int64_t off = (int64_t)pr * n + e;
    const u64 v = src[client * lay.src_client + k * lay.src_stride + off];
    u64 *dst = acc + client * lay.acc_client + k * ct_words + off;
    if (add) {
        const u64 p = c.p[pr % c.rows];
        const u64 s = *dst + v;
        *dst = s >= p ? s - p : s;
    } else {
        *dst = v;
    }
}

// acc[k] (+)= src[k * src_item_stride] for k < items; per_client > 0 splits the items into clients (AccLayout)
cudaError_t launch_accumulate(const Context &c, int l, u64 *acc, const u64 *src, int64_t src_item_stride, int64_t items,
                              bool add, cudaStream_t s, const signed char *modes = nullptr, int64_t per_client = 0,
                              int64_t src_client_stride = 0, int64_t acc_client_stride = 0) {
    const RowModuli rc = row_moduli(c, c.map_q(l));
    const AccLayout lay{per_client > 0 ? per_client : std::max<int64_t>(items, 1), src_item_stride, src_client_stride,
                        acc_client_stride};
    const int threads = coeff_threads(c.n);
    return for_each_part(items, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((c.n + threads - 1) / threads), (unsigned)(2 * l), (unsigned)chunk);
        return launch(accumulate_kernel, grid, threads, 0, s, acc, src, lay, done, rc, (int)c.n, add ? 1 : 0, modes);
    });
}

struct MaskConsts {
    int rows;
    u64 p[kMaxRows], mu_hi[kMaxRows], mu_lo[kMaxRows];
};

// ciphertextEval *= plaintextMask of CiphertextMatrix.extractDenseRow (CiphertextMatrix.swift:322-324) for every query
// row of every client of a group in one launch: item = j * rows_per_client + r,
//   y[item] = ct_eval[j * ct_count + index[r]] (.) mask_eval[r]      (Eval, canonical residues)
// ct_eval: the clients' query ciphertexts after one forward NTT (gathering after the NTT gives the values of NTT after
// gathering); mask_eval: rows_per_client x L x N.
__global__ void __launch_bounds__(256) mask_product_kernel(const u64 *__restrict__ ct_eval, const u64 *__restrict__ mask_eval,
                                                          const int *__restrict__ index, u64 *__restrict__ y,
                                                          const __grid_constant__ MaskConsts c, int n, int rows_per_client,
                                                          long long ct_count, long long item0) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int pr = blockIdx.y, row = pr % c.rows;  // poly * rows + RNS row
    const long long item = item0 + blockIdx.z, client = item / rows_per_client;
    const int r = (int)(item - client * rows_per_client);
    const long long ct_words = 2LL * c.rows * n, off = (long long)pr * n + e;
    const u64 a = ct_eval[(client * ct_count + index[r]) * ct_words + off];
    const u64 m = mask_eval[((long long)r * c.rows + row) * n + e];
    y[item * ct_words + off] = barrett128(mul_wide(a, m), c.p[row], c.mu_hi[row], c.mu_lo[row]);
}

cudaError_t launch_mask_product(const Context &c, const u64 *ct_eval, int64_t ct_count, const u64 *mask_eval, const int *index,
                                int64_t rows_per_client, int clients, u64 *y, cudaStream_t s) {
    MaskConsts mc;
    const NttRowMap map = c.map_q(c.L);
    mc.rows = c.L;
    for (int r = 0; r < c.L; ++r) {
        const ModSlot &S = c.slots[map.slot[r]].dev;
        mc.p[r] = S.p;
        mc.mu_hi[r] = S.mu_hi;
        mc.mu_lo[r] = S.mu_lo;
    }
    const int threads = coeff_threads(c.n);
    return for_each_part(rows_per_client * clients, [&](int64_t done, int64_t chunk) {
        dim3 grid((unsigned)((c.n + threads - 1) / threads), (unsigned)(2 * c.L), (unsigned)chunk);
        return launch(mask_product_kernel, grid, threads, 0, s, ct_eval, mask_eval, index, y, mc, (int)c.n, (int)rows_per_client,
                      ct_count, done);
    });
}

// GaloisElement.rotatingColumns(by:degree:) (PolyRq/Galois.swift:195-212)
unsigned rotating_columns(int step, int64_t degree) {
    unsigned positive = (unsigned)(step < 0 ? -step : step);
    if (step > 0) positive = (unsigned)(degree >> 1) - positive;
    unsigned long long g = 1, base = 3, mod = 2ull * (unsigned long long)degree;
    for (unsigned e = positive; e; e >>= 1) {
        if (e & 1) g = g * base % mod;
        base = base * base % mod;
    }
    return (unsigned)g;
}

int32_t find_key(const hecuda_evk *k, unsigned element, const u64 **key) {
    hecuda_evk *km = const_cast<hecuda_evk *>(k);
    std::lock_guard<std::mutex> g(km->mu);
    auto it = km->galois.find(element);
    if (it == km->galois.end()) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisElement: " + std::to_string(element));
    *key = it->second;
    return HECUDA_OK;
}

struct MatrixQuery {
    int32_t rows;                      // ciphertextMatrix.rowCount
    const int32_t *ciphertext_index;   // per row
    const u64 *host_masks;             // rows x N coefficient plaintexts
    const int32_t *rotate_count;       // per row
    int32_t column_step;
    const int32_t *pack_rotations;     // single rotations composing rotateColumnsMultiStep(by: matrix.rowCount)
    int32_t pack_rotation_count;
    const u64 *device_masks = nullptr;  // host_masks already on the device (the protobuf call encodes them there)
};

// What the matrix and query shapes fix: S query rows per SIMD row of a packed result, G packing groups, the ciphertexts
// of one reply, the top packing position and the longest replication chain.
struct MatrixShape {
    int64_t S, G, outputs, top;
    int32_t max_rot;
};
MatrixShape matrix_shape(const Context &c, const hecuda_pnns_matrix *m, const MatrixQuery &q) {
    MatrixShape sh;
    const int64_t R = q.rows;
    sh.S = (c.n / 2) / m->row_count;
    sh.G = sh.S > 0 ? (R + sh.S - 1) / sh.S : 0;
    sh.outputs = sh.S > 0 ? (sh.G + 1) / 2 : R * m->result_count;
    sh.top = std::min<int64_t>(sh.S, R) - 1;  // the longest group: positions above it hold nothing
    sh.max_rot = 0;
    for (int64_t r = 0; r < R && R > 1; ++r) sh.max_rot = std::max(sh.max_rot, q.rotate_count[r]);
    return sh;
}

// The key-switching keys of one client's call, found before anything is enqueued.
struct PnnsKeys {
    const u64 *rot1 = nullptr, *rotb = nullptr;  // mulTranspose(vector:): rotateColumns(by: -1), (by: -babyStep)
    const u64 *step = nullptr, *swap = nullptr;  // extractDenseRow: rotateColumns(by: column_step), swapRows
    std::vector<const u64 *> pack;              // the single rotations of rotateColumnsMultiStep(by: rowCount)
};
int32_t vector_keys(const hecuda_evk *k, int64_t n, const hecuda_pnns_matrix *m, PnnsKeys &keys) {
    int32_t rc;
    if (m->baby > 1 && (rc = find_key(k, rotating_columns(-1, n), &keys.rot1))) return rc;
    if (m->giant > 1 && (rc = find_key(k, rotating_columns(-m->baby, n), &keys.rotb))) return rc;
    return HECUDA_OK;
}
int32_t matrix_keys(const hecuda_evk *k, int64_t n, const hecuda_pnns_matrix *m, const MatrixQuery &q, const MatrixShape &sh,
                    PnnsKeys &keys) {
    int32_t rc;
    if (q.rows > 1) {
        if (sh.max_rot > 0 && (rc = find_key(k, rotating_columns(q.column_step, n), &keys.step))) return rc;
        if ((rc = find_key(k, (unsigned)(2 * n - 1), &keys.swap))) return rc;
    }
    if ((rc = vector_keys(k, n, m, keys))) return rc;
    keys.pack.assign((size_t)q.pack_rotation_count, nullptr);
    for (int32_t i = 0; i < q.pack_rotation_count && sh.S > 1; ++i)
        if ((rc = find_key(k, rotating_columns(q.pack_rotations[i], n), &keys.pack[(size_t)i]))) return rc;
    return HECUDA_OK;
}

// One rotation's keys for a group: client j's pick(keys[j]) for its per_client consecutive items
template <class Pick>
KsKeyTable key_table(const PnnsKeys *keys, int clients, int64_t per_client, Pick pick) {
    KsKeyTable t{};
    for (int j = 0; j < clients; ++j) t.key[j] = pick(keys[j]);
    t.items_per_client = per_client;
    return t;
}

// batched applyGalois over `items` contiguous ciphertexts, chunked by the scratch size; with clients > 1 every
// launch switches each client's items with the client's key (table)
int32_t galois_batch(const Context &c, u64 *scratch, int64_t chunk, KsKeyTable table, int clients, unsigned element,
                     const u64 *in, u64 *out, int64_t items, cudaStream_t s) {
    const size_t ct_words = (size_t)2 * c.L * c.n;
    for (int64_t done = 0; done < items; done += chunk) {
        const int64_t part = std::min<int64_t>(chunk, items - done);
        table.item0 = done;
        cudaError_t e = apply_galois_chunk(c, scratch, table.key[0], in + ct_words * done, c.L, element, out + ct_words * done,
                                           part, s, clients > 1 ? &table : nullptr);
        if (e != cudaSuccess) return cuda_fail(e, "applyGalois");
    }
    return HECUDA_OK;
}

// PlaintextMatrix.mulTranspose(vector:using:) for `clients` clients' `batch` query vectors each: d_vec = clients x batch
// ciphertexts (Coeff), client j with keys[j]; d_out = clients x batch x results ciphertexts.  Every stage is one pass
// over all the vectors; a single client issues the single-client launches (one scan per vector).
int32_t mul_transpose_device(const hecuda_context *h, const PnnsKeys *keys, int clients, const hecuda_pnns_matrix *m,
                             const u64 *d_vec, int64_t batch, bool to_single, u64 *d_out, cudaStream_t s) {
    const Context &c = *h->ctx;
    const int L = c.L;
    const int64_t n = c.n;
    const size_t ct_words = (size_t)2 * L * n;
    const int baby = m->baby, giant = m->giant;
    const int64_t results = m->result_count, vectors = batch * clients;
    const unsigned e1 = n > 2 ? rotating_columns(-1, n) : 0, eb = rotating_columns(-baby, n);
    int32_t rc;
    StreamBuffers tmp(s);
    u64 *states = nullptr, *rotated = nullptr, *ip = nullptr, *acc[2] = {nullptr, nullptr}, *scratch = nullptr, *ms = nullptr;
    const int64_t gal_items = std::max<int64_t>(batch, batch * results);
    // items per applyGalois pass: grows with the number of clients, so the launch count does not
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, gal_items)) * clients;
    CK(tmp.alloc(&states, ct_words * baby * vectors));
    CK(tmp.alloc(&rotated, ct_words * baby * vectors));
    CK(tmp.alloc(&ip, ct_words * results * giant * vectors));
    CK(tmp.alloc(&acc[0], ct_words * results * vectors));
    CK(tmp.alloc(&acc[1], ct_words * results * vectors));
    CK(tmp.alloc(&scratch, galois_scratch_words(c, L) * (size_t)chunk));
    CK(tmp.alloc(&ms, ct_words * results * vectors));
    cudaError_t e;
    // 1) v_j = theta^j(v): states[j][vector]                                (MatrixMultiplication.swift:180-189)
    CK(cudaMemcpyAsync(states, d_vec, ct_words * vectors * sizeof(u64), cudaMemcpyDeviceToDevice, s));
    const KsKeyTable key1 = key_table(keys, clients, batch, [](const PnnsKeys &k) { return k.rot1; });
    for (int j = 1; j < baby; ++j)
        if ((rc = galois_batch(c, scratch, chunk, key1, clients, e1, states + ct_words * (j - 1) * vectors,
                               states + ct_words * j * vectors, vectors, s)))
            return rc;
    // convertToEvalFormat (:190-193), then [j][vector] -> [vector][j] so that each vector's states are consecutive
    const NttRowMap map = c.map_q(L);
    if ((e = launch_ntt_forward(c, map, states, states, (int64_t)baby * vectors * 2 * L, s)) != cudaSuccess) return cuda_fail(e, "ntt");
    if (vectors == 1) {
        std::swap(states, rotated);
    } else {
        for (int j = 0; j < baby; ++j)
            CK(cudaMemcpy2DAsync(rotated + ct_words * j, ct_words * baby * sizeof(u64), states + ct_words * j * vectors,
                                 ct_words * sizeof(u64), ct_words * sizeof(u64), (size_t)vectors, cudaMemcpyDeviceToDevice, s));
    }
    // 2) w_k: one inner product per (result ciphertext, giant step)                         (:197-216)
    if (clients == 1) {
        for (int64_t b = 0; b < batch; ++b)
            if ((e = launch_inner_product_plain(c, rotated + ct_words * baby * b, 2, L, baby, m->d_plain, m->d_present,
                                                ip + ct_words * results * giant * b, results * giant, s)) != cudaSuccess)
                return cuda_fail(e, "innerProduct(ciphertexts:plaintexts:)");
    } else {  // the matrix streams once for the group: each vector's rotated states are one "client" of the scan
        if ((e = launch_inner_product_plain_clients(c, rotated, (int64_t)ct_words * baby, (int)vectors, L, baby, m->d_plain,
                                                    nullptr, m->d_present, ip, (int64_t)ct_words * results * giant,
                                                    results * giant, s)) != cudaSuccess)
            return cuda_fail(e, "innerProduct(ciphertexts:plaintexts:)");
    }
    if ((e = launch_ntt_inverse(c, map, ip, ip, vectors * results * giant * 2 * L, kScalePlain, s)) != cudaSuccess)
        return cuda_fail(e, "ntt");
    // 3) rotateColumnsAndSum(by: -babyStep): Horner over the giant steps, all (vector, result) pairs at once (:218-226)
    const int64_t items = vectors * results;
    const KsKeyTable keyb = key_table(keys, clients, batch * results, [](const PnnsKeys &k) { return k.rotb; });
    int cur = 0;
    if ((e = launch_accumulate(c, L, acc[cur], ip + ct_words * (giant - 1), (int64_t)ct_words * giant, items, false, s)) != cudaSuccess)
        return cuda_fail(e, "sum");
    for (int g = giant - 2; g >= 0; --g) {
        if ((rc = galois_batch(c, scratch, chunk, keyb, clients, eb, acc[cur], acc[cur ^ 1], items, s))) return rc;
        cur ^= 1;
        if ((e = launch_accumulate(c, L, acc[cur], ip + ct_words * g, (int64_t)ct_words * giant, items, true, s)) != cudaSuccess)
            return cuda_fail(e, "sum");
    }
    // Server.computeResponse: modSwitchDownToSingle (Server.swift:79-80)
    if (!to_single || L == 1) {
        CK(cudaMemcpyAsync(d_out, acc[cur], ct_words * items * sizeof(u64), cudaMemcpyDeviceToDevice, s));
        return HECUDA_OK;
    }
    const u64 *src = acc[cur];
    for (int l = L; l > 1; --l) {
        u64 *dst = l == 2 ? d_out : (src == ms ? acc[cur] : ms);
        if ((e = launch_mod_switch(c, src, l, dst, items * 2, s)) != cudaSuccess) return cuda_fail(e, "modSwitchDown");
        src = dst;
    }
    return HECUDA_OK;
}

// PlaintextMatrix.mulTranspose(matrix:using:) (MatrixMultiplication.swift:236-298) with CiphertextMatrix.extractDenseRow
// (CiphertextMatrix.swift:245-352) batched over all query rows, for `clients` clients' queries of the same shape:
// d_cts = clients x ct_count ciphertexts (Coeff), client j with keys[j]; d_out = clients x outputs ciphertexts.
int32_t mul_transpose_matrix_device(const hecuda_context *h, const PnnsKeys *keys, int clients, const hecuda_pnns_matrix *m,
                                    const u64 *d_cts, int64_t ct_count, const MatrixQuery &q, bool to_single, u64 *d_out,
                                    cudaStream_t s) {
    const Context &c = *h->ctx;
    const int L = c.L;
    const int64_t n = c.n, R = q.rows, results = m->result_count, rows = R * clients;
    const size_t ct_words = (size_t)2 * L * n;
    const MatrixShape sh = matrix_shape(c, m, q);
    const int64_t S = sh.S, G = sh.G, outputs = sh.outputs, top = sh.top;
    StreamBuffers tmp(s);
    const int64_t per_client_chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, R)), chunk = per_client_chunk * clients;
    u64 *x = nullptr, *y = nullptr, *z = nullptr, *scratch = nullptr, *inner = nullptr, *masks = nullptr, *mask_eval = nullptr;
    signed char *d_modes = nullptr;
    CK(tmp.alloc(&x, ct_words * rows));
    CK(tmp.alloc(&y, ct_words * rows));
    CK(tmp.alloc(&z, ct_words * rows));
    CK(tmp.alloc(&scratch, galois_scratch_words(c, L) * (size_t)chunk));
    CK(tmp.alloc(&inner, ct_words * rows * results));
    const NttRowMap map = c.map_q(L);
    const unsigned swap_element = (unsigned)(2 * n - 1);
    cudaError_t e;
    int32_t rc;
    // mode tables, one row of the group's items per step: replication steps (extractDenseRow) then packing positions
    std::vector<signed char> modes;
    for (int32_t t = 1; t <= sh.max_rot; ++t)
        for (int j = 0; j < clients; ++j)
            for (int64_t r = 0; r < R; ++r) modes.push_back(t <= q.rotate_count[r] ? 2 : 0);
    const size_t pack_modes_offset = modes.size();
    for (int64_t p = top; p >= 0 && S > 0; --p)
        for (int j = 0; j < clients; ++j)
            for (int64_t g = 0; g < G; ++g) {
                const int64_t size = std::min<int64_t>(S, R - g * S);
                modes.push_back(p == size - 1 ? 1 : (p < size - 1 ? 2 : 0));
            }
    CK(tmp.alloc_bytes((void **)&d_modes, modes.size()));
    if (!modes.empty()) CK(cudaMemcpyAsync(d_modes, modes.data(), modes.size(), cudaMemcpyHostToDevice, s));
    if (R == 1) {  // extractDenseRow is the identity for a single row (:263-265)
        CK(cudaMemcpy2DAsync(y, ct_words * sizeof(u64), d_cts, ct_words * ct_count * sizeof(u64), ct_words * sizeof(u64),
                             (size_t)clients, cudaMemcpyDeviceToDevice, s));
    } else {
        const unsigned step_element = rotating_columns(q.column_step, n);
        CK(tmp.alloc(&mask_eval, (size_t)L * n * R));
        if (q.device_masks) {
            masks = const_cast<u64 *>(q.device_masks);
        } else {
            CK(tmp.alloc(&masks, (size_t)n * R));
            CK(cudaMemcpyAsync(masks, q.host_masks, (size_t)n * R * sizeof(u64), cudaMemcpyHostToDevice, s));
        }
        // ciphertextEval *= plaintextMask (:322-324)
        if (clients == 1) {
            for (int64_t r = 0; r < R; ++r)
                CK(cudaMemcpyAsync(x + ct_words * r, d_cts + ct_words * q.ciphertext_index[r], ct_words * sizeof(u64),
                                   cudaMemcpyDeviceToDevice, s));
            if ((e = launch_ntt_forward(c, map, x, x, R * 2 * L, s)) != cudaSuccess) return cuda_fail(e, "ntt");
            if ((e = launch_plaintext_to_eval(c, masks, L, mask_eval, R, s)) != cudaSuccess) return cuda_fail(e, "plaintext_to_eval");
            for (int64_t r = 0; r < R; ++r)
                if ((e = launch_inner_product_plain(c, x + ct_words * r, 2, L, 1, mask_eval + (size_t)L * n * r, nullptr,
                                                    y + ct_words * r, 1, s)) != cudaSuccess)
                    return cuda_fail(e, "multiply by mask");
        } else {  // each client's query ciphertexts through one forward NTT, then every row's product in one launch
            u64 *ct_eval = nullptr;
            int *d_index = nullptr;
            CK(tmp.alloc(&ct_eval, ct_words * ct_count * clients));
            CK(tmp.alloc_bytes((void **)&d_index, sizeof(int) * (size_t)R));
            CK(cudaMemcpyAsync(d_index, q.ciphertext_index, sizeof(int) * (size_t)R, cudaMemcpyHostToDevice, s));
            if ((e = launch_ntt_forward(c, map, d_cts, ct_eval, ct_count * clients * 2 * L, s)) != cudaSuccess) return cuda_fail(e, "ntt");
            if ((e = launch_plaintext_to_eval(c, masks, L, mask_eval, R, s)) != cudaSuccess) return cuda_fail(e, "plaintext_to_eval");
            if ((e = launch_mask_product(c, ct_eval, ct_count, mask_eval, d_index, R, clients, y, s)) != cudaSuccess)
                return cuda_fail(e, "multiply by mask");
        }
        if ((e = launch_ntt_inverse(c, map, y, y, rows * 2 * L, kScalePlain, s)) != cudaSuccess) return cuda_fail(e, "ntt");
        // replicate across one SIMD row: rotate the copy, add where the row still needs copies (:331-336)
        const KsKeyTable key_step = key_table(keys, clients, R, [](const PnnsKeys &k) { return k.step; });
        const u64 *copy = y;
        u64 *ping[2] = {x, z};
        for (int32_t t = 1; t <= sh.max_rot; ++t) {
            u64 *dst = ping[t & 1];
            if ((rc = galois_batch(c, scratch, chunk, key_step, clients, step_element, copy, dst, rows, s))) return rc;
            copy = dst;
            if ((e = launch_accumulate(c, L, y, copy, (int64_t)ct_words, rows, true, s, d_modes + (size_t)(t - 1) * rows)) != cudaSuccess)
                return cuda_fail(e, "sum");
        }
        // both SIMD rows: ciphertext += swapRows(ciphertext) (:342-345)
        const KsKeyTable key_swap = key_table(keys, clients, R, [](const PnnsKeys &k) { return k.swap; });
        if ((rc = galois_batch(c, scratch, chunk, key_swap, clients, swap_element, y, x, rows, s))) return rc;
        if ((e = launch_accumulate(c, L, y, x, (int64_t)ct_words, rows, true, s)) != cudaSuccess) return cuda_fail(e, "sum");
    }
    if ((rc = mul_transpose_device(h, keys, clients, m, y, R, false, inner, s))) return rc;
    u64 *final_cts = inner;
    if (S > 0) {  // pack the result columns (:262-283); here results == 1, so client j's products are inner[j * R ...]
        u64 *acc[2] = {x, y};
        int cur = 0;
        CK(cudaMemsetAsync(acc[0], 0, ct_words * G * clients * sizeof(u64), s));
        const int64_t gchunk = std::max<int64_t>(1, std::min<int64_t>(per_client_chunk, G)) * clients;
        size_t mode_row = pack_modes_offset;
        for (int64_t p = top; p >= 0; --p, mode_row += (size_t)(G * clients)) {
            if (p < top)
                for (int32_t i = 0; i < q.pack_rotation_count; ++i) {  // rotateColumnsMultiStep(by: dimensions.rowCount)
                    const KsKeyTable key = key_table(keys, clients, G, [i](const PnnsKeys &k) { return k.pack[(size_t)i]; });
                    if ((rc = galois_batch(c, scratch, gchunk, key, clients, rotating_columns(q.pack_rotations[i], n), acc[cur],
                                           acc[cur ^ 1], G * clients, s)))
                        return rc;
                    cur ^= 1;
                }
            if ((e = launch_accumulate(c, L, acc[cur], inner + ct_words * p, (int64_t)ct_words * S, G * clients, true, s,
                                       d_modes + mode_row, G, (int64_t)ct_words * R, (int64_t)ct_words * G)) != cudaSuccess)
                return cuda_fail(e, "sum");
        }
        // swapRowsAndAdd(swapping: packedRows[1], addingTo: packedRows[0]) for every full pair (:277-281)
        const int64_t pairs = G / 2;
        u64 *packed = z;
        if ((e = launch_accumulate(c, L, packed, acc[cur], (int64_t)ct_words * 2, outputs * clients, false, s, nullptr, outputs,
                                   (int64_t)ct_words * G, (int64_t)ct_words * outputs)) != cudaSuccess)
            return cuda_fail(e, "copy");
        if (pairs > 0) {
            u64 *odd = acc[cur ^ 1];
            if ((e = launch_accumulate(c, L, odd, acc[cur] + ct_words, (int64_t)ct_words * 2, pairs * clients, false, s, nullptr,
                                       pairs, (int64_t)ct_words * G, (int64_t)ct_words * pairs)) != cudaSuccess)
                return cuda_fail(e, "copy");
            const KsKeyTable key_swap = key_table(keys, clients, pairs, [](const PnnsKeys &k) { return k.swap; });
            if ((rc = galois_batch(c, scratch, std::max<int64_t>(1, std::min<int64_t>(per_client_chunk, pairs)) * clients, key_swap,
                                   clients, swap_element, odd, inner, pairs * clients, s)))
                return rc;
            if ((e = launch_accumulate(c, L, packed, inner, (int64_t)ct_words, pairs * clients, true, s, nullptr, pairs,
                                       (int64_t)ct_words * pairs, (int64_t)ct_words * outputs)) != cudaSuccess)
                return cuda_fail(e, "sum");
        }
        final_cts = packed;
    }
    const int64_t replies = outputs * clients;
    if (!to_single || L == 1) {
        CK(cudaMemcpyAsync(d_out, final_cts, ct_words * replies * sizeof(u64), cudaMemcpyDeviceToDevice, s));
    } else {
        const u64 *src = final_cts;
        u64 *spare[2] = {nullptr, nullptr};  // sized for the outputs (more than R ciphertexts when rowCount > N)
        CK(tmp.alloc(&spare[0], ct_words * replies));
        CK(tmp.alloc(&spare[1], ct_words * replies));
        int which = 0;
        for (int l = L; l > 1; --l) {
            u64 *dst = l == 2 ? d_out : spare[which];
            which ^= 1;
            if ((e = launch_mod_switch(c, src, l, dst, replies * 2, s)) != cudaSuccess) return cuda_fail(e, "modSwitchDown");
            src = dst;
        }
    }
    CK(cudaStreamSynchronize(s));  // `modes` and the caller's descriptor arrays are host temporaries
    return HECUDA_OK;
}

int32_t check_args(const hecuda_context *h, const hecuda_evk *k, const hecuda_pnns_matrix *m, const void *vectors,
                   int64_t batch, const void *out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!m || m->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongContext: plaintext matrix belongs to another context");
    if (!k) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (batch < 0 || (batch && (!vectors || !out))) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    return HECUDA_OK;
}

// the query-shape checks of mulTranspose(matrix:), common to the single-client and the many-clients calls
int32_t check_matrix_query(const Context &c, int32_t ciphertext_count, const MatrixQuery &q) {
    if (ciphertext_count < 1 || q.rows < 1 || q.pack_rotation_count < 0 || (q.pack_rotation_count && !q.pack_rotations))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    if (q.rows > 1) {
        if (!q.ciphertext_index || !(q.host_masks || q.device_masks) || !q.rotate_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "null row descriptors");
        if (q.column_step < 1 || q.column_step > c.n / 2) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
        for (int32_t r = 0; r < q.rows; ++r)
            if (q.ciphertext_index[r] < 0 || q.ciphertext_index[r] >= ciphertext_count || q.rotate_count[r] < 0)
                return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongCiphertextCount: row descriptor out of range");
    }
    return HECUDA_OK;
}

int32_t check_capacity(const MatrixShape &sh, int64_t out_capacity, int64_t *out_count) {
    *out_count = sh.outputs;
    if (sh.outputs > out_capacity)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "output buffer too small: needs " + std::to_string(sh.outputs) + " ciphertexts");
    return HECUDA_OK;
}

// Every client checked, and every Galois key of every client found, before anything is enqueued: a failure leaves
// `out` untouched, and its message names the client by its index in the call.
int32_t check_clients(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count, const hecuda_pnns_matrix *m,
                      const void *cts, int32_t ciphertext_count, const MatrixQuery &q, const void *out, int64_t out_capacity,
                      int64_t *out_count, std::vector<PnnsKeys> &keys) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!evks || !cts || !out || !out_count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (client_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "client_count must be at least 1");
    if (!m || m->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongContext: plaintext matrix belongs to another context");
    const Context &c = *h->ctx;
    if ((rc = check_matrix_query(c, ciphertext_count, q))) return rc;
    const MatrixShape sh = matrix_shape(c, m, q);
    if ((rc = check_capacity(sh, out_capacity, out_count))) return rc;
    keys.assign((size_t)client_count, PnnsKeys{});
    for (int32_t j = 0; j < client_count; ++j) {
        const std::string who = "client " + std::to_string(j) + ": ";
        if (!evks[j]) return fail(HECUDA_ERR_MISSING_KEY, who + "missingGaloisKey");
        if (evks[j]->owner != h)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "invalidContext: evaluation key belongs to another context");
        if ((rc = matrix_keys(evks[j], c.n, m, q, sh, keys[(size_t)j]))) return fail(rc, who + last_error_cstr());
    }
    return HECUDA_OK;
}

// Server.computeResponse for every client of a call through one workspace stream, group by group: stage a group's
// queries (words, or seeded bytes expanded on the device when `wc` is given), answer the group, copy its replies back
// (packed by `wc`).  Temporaries are sized for one group.  Reply j of client c goes to out + (c * out_capacity + j)
// replies.
int32_t respond_clients(const hecuda_context *h, const std::vector<PnnsKeys> &keys, const hecuda_pnns_matrix *m,
                        const MatrixQuery &q, int32_t ciphertext_count, int64_t outputs, const void *queries,
                        const uint8_t *query_seeds, WireCodec *wc, void *out, int64_t out_capacity) {
    const Context &c = *h->ctx;
    const int32_t client_count = (int32_t)keys.size();
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    const int group = std::min<int32_t>(HECUDA_PNNS_CLIENT_GROUP, client_count);
    const size_t query_words = (size_t)2 * c.L * c.n * ciphertext_count;
    const size_t reply_bytes = wc ? wc->reply_bytes() : (size_t)2 * c.n * sizeof(u64);
    const size_t poly0_bytes = wc ? wc->query_bytes * ciphertext_count : 0, seed_bytes = (size_t)32 * ciphertext_count;
    u64 *d_query = nullptr, *d_reply = nullptr;
    unsigned char *d_poly0 = nullptr, *d_seeds = nullptr;
    CK(tmp.alloc(&d_query, query_words * group));
    CK(tmp.alloc(&d_reply, (size_t)2 * c.n * outputs * group));
    if (wc) {
        CK(tmp.alloc_bytes((void **)&d_poly0, poly0_bytes * group));
        CK(tmp.alloc_bytes((void **)&d_seeds, seed_bytes * group));
        CK(wc->alloc(tmp, c, outputs * group));
    }
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    for (int32_t first = 0; first < client_count; first += group) {
        const int clients = std::min<int32_t>(group, client_count - first);
        if (wc) {  // Query.ciphertexts arrive as SerializedCiphertext.seeded (SerializedCiphertext.swift:41-49)
            CK(cudaMemcpyAsync(d_poly0, (const uint8_t *)queries + poly0_bytes * first, poly0_bytes * clients, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(d_seeds, query_seeds + seed_bytes * first, seed_bytes * clients, cudaMemcpyHostToDevice, s));
            cudaError_t e = expand_seeded_device(c, c.L, d_poly0, d_seeds, d_query, (int64_t)ciphertext_count * clients, s);
            if (e != cudaSuccess) return cuda_fail(e, "expand seeded query");
        } else {
            CK(cudaMemcpyAsync(d_query, (const u64 *)queries + query_words * first, query_words * clients * sizeof(u64),
                               cudaMemcpyHostToDevice, s));
        }
        int32_t rc = mul_transpose_matrix_device(h, keys.data() + first, clients, m, d_query, ciphertext_count, q, true, d_reply, s);
        if (rc) return rc;
        const void *replies = d_reply;
        if (wc) {  // ApplicationProtobuf/PnnsConversionApi.swift:48: serialized forDecryption
            if ((rc = wc->pack(c, d_reply, outputs * clients, s))) return rc;
            replies = wc->reply;
        }
        CK(cudaMemcpy2DAsync((uint8_t *)out + reply_bytes * out_capacity * first, reply_bytes * out_capacity, replies,
                             reply_bytes * outputs, reply_bytes * outputs, (size_t)clients, cudaMemcpyDeviceToHost, s));
    }
    CK(wait_stream(s));
    return HECUDA_OK;
}

// The matrix shape a .diagonal PlaintextMatrix accepts; dimension = nextPow2(column_count)
int32_t check_dimensions(const Context &c, int64_t row_count, int64_t column_count, int64_t &dimension) {
    if (row_count < 1 || column_count < 1 || column_count > c.n / 2)  // PnnsError.invalidMatrixDimensions (PlaintextMatrix.swift:429-431)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    dimension = 1;
    while (dimension < column_count) dimension <<= 1;
    return HECUDA_OK;
}

// The BabyStepGiantStep a resident matrix of padded dimension `dimension` accepts (MatrixMultiplication.swift:26-62)
int32_t check_steps(const Context &c, int64_t dimension, int32_t baby_step, int32_t giant_step) {
    if (baby_step < 1 || giant_step < 1 || baby_step < giant_step || (int64_t)baby_step * giant_step < dimension ||
        (int64_t)baby_step * (giant_step - 1) >= dimension || baby_step >= c.n / 2)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongMatrixPacking: babyStep / giantStep do not cover the padded dimension");
    return HECUDA_OK;
}

// PlaintextMatrix.init(signedValues:) + diagonalPlaintexts (PlaintextMatrix.swift:155-190, 417-482) on the default
// stream from row-major values already on the device: SIMD-encodes `count` plaintexts slab by slab (in slot order when
// `resident`), handing each slab's coefficients to sink(first, items, d_coeff).  Frees its buffers before it returns;
// HECUDA_ERR_INVALID_ARGUMENT when a value is outside centeredToRemainder's range and `reduce` is off.
template <class Sink>
int32_t pnns_encode_slabs(const Context &c, const procdb::PnnsShape &shape, const int64_t *d_values, bool reduce,
                          bool resident, int64_t count, Sink sink) {
    const int64_t slab = coefficient_slab(c);
    int *d_bad = nullptr;
    u64 *d_coeff = nullptr;
    int bad = 0;
    cudaError_t e = cudaMalloc(&d_bad, sizeof(int));
    if (e == cudaSuccess) e = fill(d_bad, 0, sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc(&d_coeff, (size_t)std::min(slab, count) * c.n * sizeof(u64));
    for (int64_t done = 0; e == cudaSuccess && done < count; done += slab) {
        const int64_t items = std::min(slab, count - done);
        e = launch_pnns_diagonal(c, shape, d_values, reduce, resident, done, items, d_coeff, d_bad, nullptr);
        if (e == cudaSuccess) e = sink(done, items, d_coeff);
    }
    if (e == cudaSuccess) e = cudaMemcpy(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(d_coeff);
    cudaFree(d_bad);
    if (e != cudaSuccess) return cuda_fail(e, "pnns diagonal packing");
    if (bad)  // Scalar.centeredToRemainder's precondition (Scalar.swift:85-87)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "signed value outside [-floor(t/2), floor((t-1)/2)]; pass reduce to reduce mod t");
    return HECUDA_OK;
}

// pnns_encode_slabs from host values: uploads them once
template <class Sink>
int32_t pnns_encode_slabs_host(const Context &c, const procdb::PnnsShape &shape, const int64_t *values, bool reduce,
                               bool resident, int64_t count, Sink sink) {
    const size_t value_bytes = (size_t)shape.rows * shape.cols * sizeof(int64_t);
    int64_t *d_values = nullptr;
    cudaError_t e = cudaMalloc(&d_values, value_bytes);
    if (e == cudaSuccess) e = upload(d_values, values, value_bytes);
    if (e != cudaSuccess) {
        cudaFree(d_values);
        return cuda_fail(e, "pnns diagonal packing");
    }
    const int32_t rc = pnns_encode_slabs(c, shape, d_values, reduce, resident, count, sink);
    cudaFree(d_values);
    return rc;
}

// The resident matrix of hecuda_pnns_matrix_create_from_values from row-major signed values on the device; the shape
// has passed check_values.  On error *out stays NULL and nothing stays allocated.
int32_t matrix_from_device_values(const hecuda_context *h, const procdb::PnnsShape &shape, const int64_t *d_values,
                                  bool reduce, hecuda_pnns_matrix **out) {
    const Context &c = *h->ctx;
    const size_t row_words = (size_t)c.L * c.n;
    const int32_t baby_step = shape.baby, giant_step = shape.giant;
    const int64_t slots = shape.results * giant_step * baby_step;
    hecuda_pnns_matrix *m = new (std::nothrow) hecuda_pnns_matrix();
    if (!m) return fail(HECUDA_ERR_CUDA, "out of host memory");
    m->owner = h;
    m->row_count = shape.rows;
    m->column_count = shape.cols;
    m->result_count = shape.results;
    m->baby = baby_step;
    m->giant = giant_step;
    m->dimension = shape.dimension;
    // slot (r, g, j) holds diagonal baby * g + j of chunk r; slots past the padded dimension are absent (all zero)
    std::vector<unsigned char> present((size_t)slots, 0);
    for (int64_t slot = 0; slot < slots; ++slot) present[(size_t)slot] = slot % ((int64_t)giant_step * baby_step) < shape.dimension;
    cudaError_t e = cudaMalloc(&m->d_plain, row_words * slots * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&m->d_present, (size_t)slots);
    if (e == cudaSuccess) e = upload(m->d_present, present.data(), (size_t)slots);
    if (e != cudaSuccess) {
        hecuda_pnns_matrix_destroy(m);
        return cuda_fail(e, "pnns matrix from values");
    }
    // Plaintext.convertToEvalFormat (MatrixMultiplication.swift:206-208), one slab of slots at a time
    int32_t rc = pnns_encode_slabs(c, shape, d_values, reduce, true, slots, [&](int64_t first, int64_t items, const u64 *d) {
        return launch_plaintext_to_eval(c, d, c.L, m->d_plain + row_words * first, items, nullptr);
    });
    if (rc == HECUDA_OK) {
        e = cudaStreamSynchronize(nullptr);
        if (e != cudaSuccess) rc = cuda_fail(e, "pnns matrix from values");
    }
    if (rc) {
        hecuda_pnns_matrix_destroy(m);
        return rc;
    }
    *out = m;
    return HECUDA_OK;
}

// resident: a matrix handle, whose baby and giant step are checked as hecuda_pnns_matrix_create checks them;
// otherwise diagonalPlaintexts, which needs only a positive baby step (giant_step is ignored)
int32_t check_values(const hecuda_context *h, const int64_t *values, int64_t row_count, int64_t column_count,
                     int32_t baby_step, int32_t giant_step, bool resident, procdb::PnnsShape &shape) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!values) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *h->ctx;
    int64_t dimension = 0;
    if ((rc = check_dimensions(c, row_count, column_count, dimension))) return rc;
    if (resident) {
        if ((rc = check_steps(c, dimension, baby_step, giant_step))) return rc;
    } else if (baby_step < 1) {
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongMatrixPacking: babyStep must be positive");
    }
    if (!c.simd) return fail(HECUDA_ERR_UNSUPPORTED, "simdEncodingNotSupported");
    shape = procdb::PnnsShape{row_count, column_count, (row_count + c.n - 1) / c.n, (int)dimension, baby_step,
                              resident ? giant_step : 1, c.logn};
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_pnns_diagonal_plaintexts(const hecuda_context *h, const int64_t *values, int32_t reduce, int64_t row_count,
                                        int64_t column_count, int32_t baby_step, uint64_t *out) {
    procdb::PnnsShape shape;
    int32_t rc = check_values(h, values, row_count, column_count, baby_step, 0, false, shape);
    if (rc) return rc;
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *h->ctx;
    return pnns_encode_slabs_host(c, shape, values, reduce != 0, false, (int64_t)shape.dimension * shape.results,
                             [&](int64_t first, int64_t items, const u64 *d) {
                                 return cudaMemcpy(out + (size_t)first * c.n, d, (size_t)items * c.n * sizeof(u64),
                                                   cudaMemcpyDeviceToHost);
                             });
}

int32_t hecuda_pnns_matrix_create_from_values(const hecuda_context *h, const int64_t *values, int32_t reduce,
                                              int64_t row_count, int64_t column_count, int32_t baby_step,
                                              int32_t giant_step, hecuda_pnns_matrix **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    procdb::PnnsShape shape;
    int32_t rc = check_values(h, values, row_count, column_count, baby_step, giant_step, true, shape);
    if (rc) return rc;
    const size_t value_bytes = (size_t)row_count * column_count * sizeof(int64_t);
    int64_t *d_values = nullptr;
    cudaError_t e = cudaMalloc(&d_values, value_bytes);
    if (e == cudaSuccess) e = upload(d_values, values, value_bytes);
    rc = e == cudaSuccess ? matrix_from_device_values(h, shape, d_values, reduce != 0, out) : cuda_fail(e, "pnns matrix from values");
    cudaFree(d_values);
    return rc;
}

int32_t hecuda_pnns_matrices_create_from_vectors(const hecuda_context *const *ctxs, int32_t plaintext_count, const float *vectors,
                                                 int64_t row_count, int64_t column_count, int64_t scaling_factor,
                                                 int32_t baby_step, int32_t giant_step, hecuda_pnns_matrix **out) {
    if (!out || !ctxs || plaintext_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument or no context");
    for (int32_t k = 0; k < plaintext_count; ++k) out[k] = nullptr;
    // For a single plaintext modulus, reduction isn't necessary (ProcessedDatabase.swift:213-214)
    const bool reduce = plaintext_count > 1;
    std::vector<procdb::PnnsShape> shapes((size_t)plaintext_count);
    int32_t rc;
    for (int32_t k = 0; k < plaintext_count; ++k) {
        // check_values only needs a non-null values pointer here; the float vectors stand in for it
        if ((rc = check_values(ctxs[k], (const int64_t *)(const void *)vectors, row_count, column_count, baby_step, giant_step,
                               true, shapes[(size_t)k])))
            return rc;
        if (ctxs[k]->ctx->n != ctxs[0]->ctx->n)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongEncryptionParameters: the contexts differ in N");
        if ((rc = check_float_vectors(vectors, row_count, column_count, scaling_factor, ctxs[k]->ctx->t, reduce, false))) return rc;
    }
    const size_t values = (size_t)row_count * column_count;
    float *d_vec = nullptr, *d_norm = nullptr;
    int64_t *d_values = nullptr;
    int *d_bad = nullptr;
    int bad = 0;
    // the float rows cross PCIe once and are normalised once; every context packs the same device-resident values
    cudaError_t e = cudaMalloc(&d_vec, values * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&d_norm, (size_t)row_count * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&d_values, values * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc(&d_bad, sizeof(int));
    if (e == cudaSuccess) e = upload(d_vec, vectors, values * sizeof(float));
    if (e == cudaSuccess) e = fill(d_bad, 0, sizeof(int));
    if (e == cudaSuccess) e = launch_pnns_normalize(d_vec, row_count, column_count, scaling_factor, d_norm, d_values, d_bad, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(d_vec);
    cudaFree(d_norm);
    cudaFree(d_bad);
    rc = e != cudaSuccess ? cuda_fail(e, "pnns vectors normalisation")
         : bad            ? fail(HECUDA_ERR_INVALID_ARGUMENT, "a vector value is not finite or a scaled value leaves Int64")
                          : HECUDA_OK;
    for (int32_t k = 0; rc == HECUDA_OK && k < plaintext_count; ++k)
        rc = matrix_from_device_values(ctxs[k], shapes[(size_t)k], d_values, reduce, &out[k]);
    cudaFree(d_values);
    if (rc)
        for (int32_t k = 0; k < plaintext_count; ++k) {
            hecuda_pnns_matrix_destroy(out[k]);
            out[k] = nullptr;
        }
    return rc;
}

int32_t hecuda_pnns_matrix_device_buffer(hecuda_pnns_matrix *m, void **device_ptr, uint64_t *bytes) {
    if (!m || !device_ptr || !bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *device_ptr = m->d_plain;
    *bytes = (uint64_t)m->result_count * m->giant * m->baby * m->owner->ctx->L * m->owner->ctx->n * sizeof(u64);
    return HECUDA_OK;
}

int32_t hecuda_pnns_matrix_present(const hecuda_pnns_matrix *m, uint8_t *out, int64_t capacity) {
    if (!m || !out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const int64_t slots = m->result_count * m->giant * m->baby;
    if (capacity < slots) return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity below the slot count");
    CK(cudaMemcpy(out, m->d_present, (size_t)slots, cudaMemcpyDeviceToHost));
    return HECUDA_OK;
}

int32_t hecuda_pnns_matrix_create(const hecuda_context *h, const uint64_t *plaintexts, int32_t eval_format,
                                  int64_t row_count, int64_t column_count, int32_t baby_step, int32_t giant_step,
                                  hecuda_pnns_matrix **out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!out || !plaintexts) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    const Context &c = *h->ctx;
    const int64_t n = c.n;
    int64_t dimension = 0;
    if ((rc = check_dimensions(c, row_count, column_count, dimension))) return rc;
    if ((rc = check_steps(c, dimension, baby_step, giant_step))) return rc;
    const int64_t results = (row_count + n - 1) / n;  // plaintextsPerColumnCount / resultCiphertextCount
    const int64_t count = dimension * results;       // PlaintextMatrix.plaintextCount, .diagonal (:269-273)
    const int64_t slots = results * giant_step * baby_step;
    const size_t row_words = (size_t)c.L * n, in_words = eval_format ? row_words : (size_t)n;
    hecuda_pnns_matrix *m = new (std::nothrow) hecuda_pnns_matrix();
    if (!m) return fail(HECUDA_ERR_CUDA, "out of host memory");
    m->owner = h;
    m->row_count = row_count;
    m->column_count = column_count;
    m->result_count = results;
    m->baby = baby_step;
    m->giant = giant_step;
    m->dimension = (int)dimension;
    std::vector<unsigned char> present((size_t)slots, 0);
    u64 *d_in = nullptr;
    cudaError_t e = cudaMalloc(&m->d_plain, row_words * slots * sizeof(u64));
    if (e == cudaSuccess) e = fill(m->d_plain, 0, row_words * slots * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&m->d_present, (size_t)slots);
    if (e == cudaSuccess) e = cudaMalloc(&d_in, in_words * count * sizeof(u64));
    if (e == cudaSuccess) e = upload(d_in, plaintexts, in_words * count * sizeof(u64));
    // plaintext index resultCount * (j + babyStep * g) + r  ->  slot (r, g, j)      (MatrixMultiplication.swift:203-205)
    for (int64_t r = 0; e == cudaSuccess && r < results; ++r)
        for (int g = 0; e == cudaSuccess && g < giant_step; ++g) {
            const int64_t terms = std::min<int64_t>(baby_step, dimension - (int64_t)baby_step * g);
            const int64_t slot = (r * giant_step + g) * baby_step;
            const u64 *src = d_in + in_words * (results * ((int64_t)baby_step * g) + r);
            if (eval_format) {
                e = cudaMemcpy2D(m->d_plain + row_words * slot, row_words * sizeof(u64), src, row_words * results * sizeof(u64),
                                 row_words * sizeof(u64), (size_t)terms, cudaMemcpyDeviceToDevice);
            } else {  // Plaintext.convertToEvalFormat per row (:206-208); gather the strided rows first
                u64 *d_rows = nullptr;
                e = cudaMalloc(&d_rows, (size_t)n * terms * sizeof(u64));
                if (e == cudaSuccess)
                    e = cudaMemcpy2D(d_rows, n * sizeof(u64), src, n * results * sizeof(u64), n * sizeof(u64), (size_t)terms,
                                     cudaMemcpyDeviceToDevice);
                if (e == cudaSuccess) e = launch_plaintext_to_eval(c, d_rows, c.L, m->d_plain + row_words * slot, terms, nullptr);
                if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
                cudaFree(d_rows);
            }
            for (int64_t j = 0; j < terms; ++j) present[(size_t)(slot + j)] = 1;
        }
    if (e == cudaSuccess) e = upload(m->d_present, present.data(), (size_t)slots);
    cudaFree(d_in);
    if (e != cudaSuccess) {
        hecuda_pnns_matrix_destroy(m);
        return cuda_fail(e, "pnns matrix upload");
    }
    *out = m;
    return HECUDA_OK;
}

int32_t hecuda_pnns_matrix_destroy(hecuda_pnns_matrix *m) {
    if (!m) return HECUDA_OK;
    if (m->d_plain) cudaFree(m->d_plain);
    if (m->d_present) cudaFree(m->d_present);
    delete m;
    return HECUDA_OK;
}

int32_t hecuda_pnns_matrix_result_count(const hecuda_pnns_matrix *m, int64_t *count) {
    if (!m || !count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *count = m->result_count;
    return HECUDA_OK;
}

int32_t hecuda_pnns_mul_transpose_vector_device(const hecuda_context *h, const hecuda_evk *k, const hecuda_pnns_matrix *m,
                                                const uint64_t *vectors, int64_t batch, int32_t mod_switch_to_single,
                                                uint64_t *out, void *stream) {
    int32_t rc = check_args(h, k, m, vectors, batch, out);
    if (rc || batch == 0) return rc;
    PnnsKeys keys;
    if ((rc = vector_keys(k, h->ctx->n, m, keys))) return rc;
    return mul_transpose_device(h, &keys, 1, m, (const u64 *)vectors, batch, mod_switch_to_single != 0, (u64 *)out,
                                (cudaStream_t)stream);
}

int32_t hecuda_pnns_mul_transpose_vector(const hecuda_context *h, const hecuda_evk *k, const hecuda_pnns_matrix *m,
                                         const uint64_t *vectors, int64_t batch, int32_t mod_switch_to_single,
                                         uint64_t *out) {
    int32_t rc = check_args(h, k, m, vectors, batch, out);
    if (rc || batch == 0) return rc;
    PnnsKeys keys;
    if ((rc = vector_keys(k, h->ctx->n, m, keys))) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const Context &c = *h->ctx;
    const size_t ct_words = (size_t)2 * c.L * c.n;
    const size_t out_words = (size_t)2 * (mod_switch_to_single ? 1 : c.L) * c.n * m->result_count * batch;
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    u64 *d_in = nullptr, *d_out = nullptr;
    CK(tmp.alloc(&d_in, ct_words * batch));
    CK(tmp.alloc(&d_out, ct_words * m->result_count * batch));
    CK(cudaMemcpyAsync(d_in, vectors, ct_words * batch * sizeof(u64), cudaMemcpyHostToDevice, s));
    rc = mul_transpose_device(h, &keys, 1, m, d_in, batch, mod_switch_to_single != 0, d_out, s);
    if (rc) {
        cudaStreamSynchronize(s);
        return rc;
    }
    CK(cudaMemcpyAsync(out, d_out, out_words * sizeof(u64), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return HECUDA_OK;
}

int32_t hecuda_pnns_mul_transpose_matrix(const hecuda_context *h, const hecuda_evk *k, const hecuda_pnns_matrix *m,
                                         const uint64_t *ciphertexts, int32_t ciphertext_count, int32_t query_row_count,
                                         const int32_t *row_ciphertext_index, const uint64_t *row_masks,
                                         const int32_t *row_rotate_count, int32_t column_step, const int32_t *pack_rotations,
                                         int32_t pack_rotation_count, int32_t mod_switch_to_single, uint64_t *out,
                                         int64_t out_capacity, int64_t *out_count) {
    int32_t rc = check_args(h, k, m, ciphertexts, ciphertext_count, out);
    if (rc) return rc;
    if (!out_count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    const Context &c = *h->ctx;
    const MatrixQuery q{query_row_count, row_ciphertext_index, (const u64 *)row_masks, row_rotate_count, column_step,
                        pack_rotations, pack_rotation_count};
    if ((rc = check_matrix_query(c, ciphertext_count, q))) return rc;
    const MatrixShape sh = matrix_shape(c, m, q);
    if ((rc = check_capacity(sh, out_capacity, out_count))) return rc;
    PnnsKeys keys;
    if ((rc = matrix_keys(k, c.n, m, q, sh, keys))) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const size_t ct_words = (size_t)2 * c.L * c.n;
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    u64 *d_in = nullptr, *d_out = nullptr;
    CK(tmp.alloc(&d_in, ct_words * ciphertext_count));
    CK(tmp.alloc(&d_out, ct_words * (size_t)std::max<int64_t>(sh.outputs, 1)));
    CK(cudaMemcpyAsync(d_in, ciphertexts, ct_words * ciphertext_count * sizeof(u64), cudaMemcpyHostToDevice, s));
    rc = mul_transpose_matrix_device(h, &keys, 1, m, d_in, ciphertext_count, q, mod_switch_to_single != 0, d_out, s);
    if (rc) {
        cudaStreamSynchronize(s);
        return rc;
    }
    const size_t out_words = (size_t)2 * (mod_switch_to_single ? 1 : c.L) * c.n * (size_t)*out_count;
    CK(cudaMemcpyAsync(out, d_out, out_words * sizeof(u64), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return HECUDA_OK;
}

int32_t hecuda_pnns_compute_response_clients(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                                             const hecuda_pnns_matrix *m, const uint64_t *ciphertexts, int32_t ciphertext_count,
                                             int32_t query_row_count, const int32_t *row_ciphertext_index,
                                             const uint64_t *row_masks, const int32_t *row_rotate_count, int32_t column_step,
                                             const int32_t *pack_rotations, int32_t pack_rotation_count, uint64_t *out,
                                             int64_t out_capacity, int64_t *out_count) {
    const MatrixQuery q{query_row_count, row_ciphertext_index, (const u64 *)row_masks, row_rotate_count, column_step,
                        pack_rotations, pack_rotation_count};
    std::vector<PnnsKeys> keys;
    int32_t rc = check_clients(h, evks, client_count, m, ciphertexts, ciphertext_count, q, out, out_capacity, out_count, keys);
    if (rc) return rc;
    return respond_clients(h, keys, m, q, ciphertext_count, *out_count, ciphertexts, nullptr, nullptr, out, out_capacity);
}

int32_t hecuda_pnns_compute_response_clients_wire(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                                                  const hecuda_pnns_matrix *m, const uint8_t *query_poly0,
                                                  const uint8_t *query_seeds, int32_t ciphertext_count, int32_t query_row_count,
                                                  const int32_t *row_ciphertext_index, const uint64_t *row_masks,
                                                  const int32_t *row_rotate_count, int32_t column_step,
                                                  const int32_t *pack_rotations, int32_t pack_rotation_count,
                                                  int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint8_t *out,
                                                  int64_t out_capacity, int64_t *out_count) {
    const MatrixQuery q{query_row_count, row_ciphertext_index, (const u64 *)row_masks, row_rotate_count, column_step,
                        pack_rotations, pack_rotation_count};
    std::vector<PnnsKeys> keys;
    int32_t rc = check_clients(h, evks, client_count, m, query_poly0, ciphertext_count, q, out, out_capacity, out_count, keys);
    if (rc) return rc;
    if (!query_seeds) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    WireCodec wc;
    if ((rc = wc.setup(*h->ctx, skip_lsbs_poly0, skip_lsbs_poly1))) return rc;
    return respond_clients(h, keys, m, q, ciphertext_count, *out_count, query_poly0, query_seeds, &wc, out, out_capacity);
}

}  // extern "C"

// ---------------------------------------------------------------- protobuf messages in and out
// PNNSRequest in, PNNSShardResponse out (pnns_proto.hpp), the query plan derived here (pnns_plan.hpp).  The device
// path is respond_clients' with the messages read in place, as the PIR protobuf path does (proto_respond.hpp).
#include "pnns_plan.hpp"
#include "pnns_proto.hpp"
#include "proto_respond.hpp"

namespace {

// The response of one call: per context its reply codec (Bfv.skipLSBsForDecryption of its t), the replies per client
// and the PNNSShardResponse layout
struct ShardReply {
    std::vector<WireCodec> wc;
    int64_t outputs = 0;
    pnnsproto::ShardLayout layout;
};
int32_t shard_reply(const hecuda_context *const *ctxs, int32_t count, const hecuda_pnns_matrix *const *ms, int64_t query_rows,
                    const uint64_t *ids, int64_t id_count, const uint8_t *metadata, const uint64_t *metadata_offsets,
                    int64_t metadata_count, ShardReply &r) {
    if (!ctxs || !ms || count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (id_count < 0 || metadata_count < 0 || (id_count && !ids) || (metadata_count && !metadata_offsets))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    for (int64_t i = 0; i < metadata_count; ++i)
        if (metadata_offsets[i + 1] < metadata_offsets[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "metadata offsets decrease");
    if (metadata_count && metadata_offsets[metadata_count] > metadata_offsets[0] && !metadata)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (query_rows < 1 || query_rows > 0xffffffffLL) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions");
    std::vector<std::array<long long, 2>> bytes;
    std::vector<std::array<int, 2>> skips;
    r.wc.assign((size_t)count, WireCodec{});
    for (int32_t k = 0; k < count; ++k) {
        int32_t rc = check_ctx(ctxs[k]);
        if (rc) return rc;
        if (!ms[k] || ms[k]->owner != ctxs[k])
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongContext: plaintext matrix " + std::to_string(k) + " belongs to another context");
        if (ms[k]->row_count != ms[0]->row_count || ms[k]->column_count != ms[0]->column_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidMatrixDimensions: the plaintext matrices differ in shape");
        const Context &c = *ctxs[k]->ctx;
        int skip[2];
        pnnsproto::skip_lsbs_for_decryption(c.q[0], c.t, c.n, skip);
        if ((rc = r.wc[(size_t)k].setup(c, skip[0], skip[1]))) return rc;
        bytes.push_back({(long long)r.wc[(size_t)k].bytes[0], (long long)r.wc[(size_t)k].bytes[1]});
        skips.push_back({skip[0], skip[1]});
    }
    // matrix_shape: S query rows per SIMD row, G packing groups; one reply per pair of groups, or per (row, result)
    const Context &c = *ctxs[0]->ctx;
    const int64_t S = (c.n / 2) / ms[0]->row_count, G = S > 0 ? (query_rows + S - 1) / S : 0;
    r.outputs = S > 0 ? (G + 1) / 2 : query_rows * ms[0]->result_count;
    r.layout = pnnsproto::place_shard_response(bytes, skips, r.outputs, (uint64_t)ms[0]->row_count, (uint64_t)query_rows, ids,
                                               id_count, metadata, metadata_offsets, metadata_count);
    return HECUDA_OK;
}

// respond_clients with PNNSRequest messages in and PNNSShardResponse messages out.  Per group: the group's messages
// uploaded back to back; per context the seeded expansion reading them in place (and the .full ciphertexts loaded over
// theirs), the group's responses and one packing launch per reply poly into the clients' messages; the framing of
// every message in one launch (before the packing, which writes between its runs); one download.
int32_t respond_proto(const hecuda_context *const *ctxs, int32_t count, const hecuda_pnns_matrix *const *ms,
                      int32_t client_count, const uint8_t *const *messages, const uint64_t *message_byte_counts,
                      const std::vector<std::vector<pnnsproto::Matrix>> &queries, const std::vector<pnnsplan::QueryPlan> &plans,
                      std::vector<MatrixQuery> &qs, const std::vector<std::vector<PnnsKeys>> &keys, const ShardReply &r,
                      uint8_t *out) {
    const hecuda_context *h = ctxs[0];
    const pnnsproto::ShardLayout &sl = r.layout;
    const int group = std::min<int32_t>(HECUDA_PNNS_CLIENT_GROUP, client_count);
    const int64_t outputs = r.outputs, R = plans[0].rows, cts = plans[0].ciphertexts;
    size_t msg_bytes = 0, ct_words = 0;
    for (int32_t first = 0; first < client_count; first += group) {
        size_t bytes = 0;
        for (int32_t j = first; j < std::min<int32_t>(first + group, client_count); ++j) bytes += message_byte_counts[j];
        msg_bytes = std::max(msg_bytes, bytes);
    }
    for (int32_t k = 0; k < count; ++k) ct_words = std::max(ct_words, (size_t)2 * ctxs[k]->ctx->L * ctxs[k]->ctx->n);
    FrameRuns frame;
    frame.size = sl.size;
    sl.frame([&](long long at, const pnnsproto::Bytes &b) { frame.put(at, b); });
    // reply ciphertext i of a group (client-major) is polys 2i, 2i + 1 of the group's responses; on context k its poly p
    // goes to byte tag[i] of the group's messages
    const size_t span = (size_t)group * outputs + 1;
    std::vector<long long> pack((size_t)count * 4 * span);
    for (int32_t k = 0; k < count; ++k)
        for (int p = 0; p < 2; ++p) {
            long long *tag = pack.data() + ((size_t)k * 2 + p) * 2 * span, *slot = tag + span;
            for (int64_t i = 0; i < group * outputs; ++i) {
                tag[i] = (i / outputs) * sl.size + sl.poly_at((size_t)k, i % outputs, p);
                slot[i] = 2 * i + p;
            }
            tag[span - 1] = group * sl.size;
        }
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    unsigned char *d_msg = nullptr, *d_out = nullptr, *d_frame = nullptr;
    u64 *d_query = nullptr, *d_resp = nullptr, *d_values = nullptr, *d_masks = nullptr;
    long long *d_pack = nullptr, *d_tables = nullptr, *d_runs = nullptr;
    const size_t table_words = (size_t)2 * cts * group + 1 + (size_t)6 * cts * group;
    const int64_t n = ctxs[0]->ctx->n;
    CK(tmp.alloc_bytes((void **)&d_msg, msg_bytes + 32));  // + 32 zero bytes: the seed a .full ciphertext expands
    CK(tmp.alloc(&d_query, ct_words * cts * group));
    CK(tmp.alloc(&d_resp, (size_t)2 * n * outputs * group));
    CK(tmp.alloc_bytes((void **)&d_out, (size_t)sl.size * group));
    CK(tmp.alloc_bytes((void **)&d_pack, pack.size() * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_tables, table_words * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_runs, frame.table.size() * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_frame, frame.bytes.size()));
    if (R > 1) {
        CK(tmp.alloc(&d_values, (size_t)R * n));
        CK(tmp.alloc(&d_masks, (size_t)count * R * n));
    }
    CodecConsts full_cc;
    std::string err;
    std::vector<std::vector<long long>> staged;  // host tables stay alive until the stream is drained
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    CK(cudaMemcpyAsync(d_pack, pack.data(), pack.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_runs, frame.table.data(), frame.table.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_frame, frame.bytes.data(), frame.bytes.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(d_msg + msg_bytes, 0, 32, s));
    cudaError_t e;
    for (int32_t k = 0; k < count && R > 1; ++k) {  // extractDenseRow's masks, SIMD-encoded once per context
        CK(cudaMemcpyAsync(d_values, plans[(size_t)k].mask_values.data(), (size_t)R * n * sizeof(u64), cudaMemcpyHostToDevice, s));
        u64 *masks = d_masks + (size_t)k * R * n;
        if ((e = launch_encode_simd(*ctxs[k]->ctx, d_values, (int)n, 0, masks, nullptr, R, s)) != cudaSuccess)
            return cuda_fail(e, "encode masks");
        qs[(size_t)k].device_masks = masks;
    }
    for (int32_t first = 0; first < client_count; first += group) {
        const int clients = std::min<int32_t>(group, client_count - first);
        std::vector<long long> msg_at((size_t)clients);
        long long at = 0;
        for (int j = 0; j < clients; ++j) {
            msg_at[(size_t)j] = at;
            CK(cudaMemcpyAsync(d_msg + at, messages[first + j], message_byte_counts[first + j], cudaMemcpyHostToDevice, s));
            at += (long long)message_byte_counts[first + j];
        }
        if ((e = launch_frame_runs(d_out, clients, sl.size, d_runs, frame.runs(), d_frame, s)) != cudaSuccess)
            return cuda_fail(e, "frame response");
        for (int32_t k = 0; k < count; ++k) {
            const Context &c = *ctxs[k]->ctx;
            std::vector<const std::vector<pnnsproto::Ciphertext> *> cts_of((size_t)clients);
            for (int j = 0; j < clients; ++j) cts_of[(size_t)j] = &queries[(size_t)(first + j)][(size_t)k].cts;
            const GroupTables t = group_tables(cts_of, msg_at, (long long)msg_bytes);
            staged.emplace_back(t.tag);
            std::vector<long long> &flat = staged.back();
            flat.insert(flat.end(), t.seed.begin(), t.seed.end());
            for (const auto &f : t.full) flat.insert(flat.end(), f.second.begin(), f.second.end());
            CK(cudaMemcpyAsync(d_tables, flat.data(), flat.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
            PolyLayout seeded;
            seeded.tag = d_tables, seeded.seed = d_tables + t.tag.size(), seeded.frame = 0;
            const int64_t batch = cts * clients;
            if ((e = expand_seeded_device(c, c.L, d_msg, nullptr, d_query, batch, s, seeded)) != cudaSuccess)
                return cuda_fail(e, "expand seeded query");
            // .full query ciphertexts (Ciphertext(deserialize:) of .full): both polys over the zero rows expanded above
            const long long *table = seeded.seed + t.seed.size();
            for (const auto &f : t.full) {
                const int64_t full = (int64_t)(f.second.size() - 1) / 2;
                if (!codec_consts(c, c.map_q(c.L), f.first, full_cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
                PolyLayout layout;
                layout.tag = table, layout.slot = table + full + 1, layout.frame = 0;
                if ((e = launch_poly_load(c, full_cc, f.first, d_msg, d_query, full, s, layout)) != cudaSuccess)
                    return cuda_fail(e, "load full query ciphertexts");
                table += f.second.size();
            }
            int32_t rc = mul_transpose_matrix_device(ctxs[k], keys[(size_t)k].data() + first, clients, ms[k], d_query, cts,
                                                     qs[(size_t)k], true, d_resp, s);
            if (rc) return rc;
            const WireCodec &wc = r.wc[(size_t)k];
            for (int p = 0; p < 2; ++p) {
                PolyLayout to;
                to.tag = d_pack + ((size_t)k * 2 + p) * 2 * span, to.slot = to.tag + span, to.frame = 0;
                if ((e = launch_poly_serialize(c, wc.out[p], wc.skip[p], d_resp, d_out, outputs * clients, s, to)) != cudaSuccess)
                    return cuda_fail(e, "serialize response");
            }
        }
        CK(cudaMemcpyAsync(out + (size_t)sl.size * first, d_out, (size_t)sl.size * clients, cudaMemcpyDeviceToHost, s));
    }
    CK(wait_stream(s));
    return HECUDA_OK;
}

// The Galois elements a client's key holds (GaloisElement.stepsFor's input for the packing plan)
std::set<uint64_t> galois_elements(const hecuda_evk *k) {
    hecuda_evk *km = const_cast<hecuda_evk *>(k);
    std::lock_guard<std::mutex> g(km->mu);
    std::set<uint64_t> out;
    for (const auto &e : km->galois) out.insert(e.first);
    return out;
}

}  // namespace

extern "C" {

int32_t hecuda_pnns_shard_response_byte_count(const hecuda_context *const *ctxs, int32_t count,
                                              const hecuda_pnns_matrix *const *matrices, int32_t query_row_count,
                                              const uint64_t *entry_ids, int64_t id_count, const uint8_t *metadata,
                                              const uint64_t *metadata_offsets, int64_t metadata_count, uint64_t *bytes) {
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    ShardReply r;
    int32_t rc = shard_reply(ctxs, count, matrices, query_row_count, entry_ids, id_count, metadata, metadata_offsets,
                             metadata_count, r);
    if (rc) return rc;
    *bytes = (uint64_t)r.layout.size;
    return HECUDA_OK;
}

int32_t hecuda_pnns_compute_response_clients_proto(const hecuda_context *const *ctxs, int32_t count,
                                                   const hecuda_evk *const *evks, int32_t client_count,
                                                   const hecuda_pnns_matrix *const *matrices,
                                                   const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                   const uint64_t *entry_ids, int64_t id_count, const uint8_t *metadata,
                                                   const uint64_t *metadata_offsets, int64_t metadata_count, uint8_t *out) {
    if (!ctxs || count < 1 || !matrices || !evks || !messages || !message_byte_counts || !out)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (client_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "client_count must be at least 1");
    int32_t rc;
    std::vector<pnnsproto::PolySizes> sizes((size_t)count);
    for (int32_t k = 0; k < count; ++k) {
        if ((rc = check_ctx(ctxs[k]))) return rc;
        if (!matrices[k] || matrices[k]->owner != ctxs[k])
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongContext: plaintext matrix " + std::to_string(k) + " belongs to another context");
        const Context &c = *ctxs[k]->ctx;
        CodecConsts qc;
        std::string err;
        if (!codec_consts(c, c.map_q(c.L), 0, qc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
        sizes[(size_t)k] = pnnsproto::poly_sizes(qc, c.n);
    }
    // every client's request walked and checked against the database, and against client 0's shape
    std::vector<std::vector<pnnsproto::Matrix>> queries((size_t)client_count);
    for (int32_t j = 0; j < client_count; ++j) {
        const std::string who = "client " + std::to_string(j) + ": ";
        if (!messages[j] && message_byte_counts[j]) return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "null argument");
        pnnsproto::Error e;
        pnnsproto::Request req;
        if (!pnnsproto::walk_pnns_request(messages[j], (long long)message_byte_counts[j], req, e) ||
            !pnnsproto::walk_query(messages[j], req, sizes, (uint64_t)matrices[0]->column_count, queries[(size_t)j], e))
            return fail(e.code, who + e.what);
        if (queries[(size_t)j][0].rows != queries[0][0].rows)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "invalidMatrixDimensions: a query of " +
                                                         std::to_string(queries[(size_t)j][0].rows) + " rows, client 0's has " +
                                                         std::to_string(queries[0][0].rows));
    }
    const int64_t R = (int64_t)queries[0][0].rows;
    ShardReply reply;
    if ((rc = shard_reply(ctxs, count, matrices, R, entry_ids, id_count, metadata, metadata_offsets, metadata_count, reply)))
        return rc;
    // keys: any context of the same N, word size and coefficient moduli (EvaluationKey.forContext's test), read in place
    for (int32_t j = 0; j < client_count; ++j) {
        const std::string who = "client " + std::to_string(j) + ": ";
        if (!evks[j]) return fail(HECUDA_ERR_MISSING_KEY, who + "missingGaloisKey");
        if (!evks[j]->owner) return fail(HECUDA_ERR_MISSING_KEY, who + "null evaluation key");
        const Context &a = *evks[j]->owner->ctx;
        for (int32_t k = 0; k < count; ++k) {
            const Context &b = *ctxs[k]->ctx;
            if (a.n != b.n || a.word_bits != b.word_bits || a.q != b.q || a.q_ks != b.q_ks)
                return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "invalidContext: the key's context differs from context " +
                                                             std::to_string(k) + " in N, word size or coefficient moduli");
        }
    }
    // the query plan, once per call, from the shape and client 0's Galois elements; every key of every client found
    const std::set<uint64_t> elements = galois_elements(evks[0]);
    std::vector<pnnsplan::QueryPlan> plans((size_t)count);
    std::vector<MatrixQuery> qs;
    std::vector<std::vector<PnnsKeys>> keys((size_t)count, std::vector<PnnsKeys>((size_t)client_count));
    for (int32_t k = 0; k < count; ++k) {
        const Context &c = *ctxs[k]->ctx;
        pnnsplan::QueryPlan &p = plans[(size_t)k];
        std::string err;
        if (!pnnsplan::plan_query(c.n, R, matrices[k]->column_count, matrices[k]->row_count, elements, p, err))
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "client 0: " + err);
        // the masks are encoded on the device by respond_proto (device_masks); the plan is in range by construction
        qs.push_back(MatrixQuery{p.rows, p.index.data(), nullptr, p.rotate.data(), p.column_step, p.pack.data(),
                                 (int32_t)p.pack.size()});
        const MatrixShape sh = matrix_shape(c, matrices[k], qs.back());
        for (int32_t j = 0; j < client_count; ++j)
            if ((rc = matrix_keys(evks[j], c.n, matrices[k], qs.back(), sh, keys[(size_t)k][(size_t)j])))
                return fail(rc, "client " + std::to_string(j) + ": " + last_error_cstr());
    }
    return respond_proto(ctxs, count, matrices, client_count, messages, message_byte_counts, queries, plans, qs, keys, reply, out);
}

}  // extern "C"

// ---------------------------------------------------------------- saving and loading processed databases
// SerializedProcessedDatabase (ProcessedDatabase.swift:56-88, PnnsConversion.swift).  The host walks or places the
// protobuf framing (pnns_database_io.hpp); whole plaintexts then cross PCIe in chunks of at most one 64 MB slab
// through the two-workspace pipeline of the PIR files (pir.cu), and the codec kernels (codec.cu) unpack each plaintext
// straight into its resident slot, or pack it from there together with its framing.
#include "database_io.hpp"
#include "pnns_database_io.hpp"

namespace {

int32_t io_fail(const pnnsio::Error &e) { return fail(e.code, e.what); }

std::string moduli_text(const std::vector<u64> &m) {
    std::string s = "[";
    for (size_t k = 0; k < m.size(); ++k) s += (k ? ", " : "") + std::to_string(m[k]);
    return s + "]";
}

// ServerConfig.validateContexts (Config.swift:125-135): one context per plaintext modulus, each with the config's
// degree, coefficient moduli (the key-switching one included) and its plaintext modulus
int32_t validate_contexts(const hecuda_context *const *ctxs, int32_t count, const hecuda_pnns_server_config &cfg) {
    const int32_t expected = 1 + cfg.extra_plaintext_moduli_count;
    if (count != expected)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongContextsCount(got: " + std::to_string(count) + ", expected: " +
                                                     std::to_string(expected) + ")");
    const std::vector<u64> want(cfg.coefficient_moduli, cfg.coefficient_moduli + cfg.coefficient_moduli_count);
    for (int32_t k = 0; k < count; ++k) {
        int32_t rc = check_ctx(ctxs[k]);
        if (rc) return rc;
        const Context &c = *ctxs[k]->ctx;
        std::vector<u64> got = c.q;
        if (c.has_ks) got.push_back(c.q_ks);
        const u64 t = k ? cfg.extra_plaintext_moduli[k - 1] : cfg.plaintext_modulus;
        if ((u64)c.n != cfg.poly_degree || c.t != t || got != want)
            return fail(HECUDA_ERR_INVALID_ARGUMENT,
                        "wrongEncryptionParameters(context " + std::to_string(k) + ": got N = " + std::to_string(c.n) +
                            ", t = " + std::to_string(c.t) + ", moduli " + moduli_text(got) + "; expected N = " +
                            std::to_string(cfg.poly_degree) + ", t = " + std::to_string(t) + ", moduli " + moduli_text(want) + ")");
    }
    return HECUDA_OK;
}

// A resident .diagonal matrix's shape, as hecuda_pnns_matrix_create checks it
struct DiagonalShape {
    int64_t dimension = 0, results = 0, count = 0, slots = 0;
    int32_t baby = 0, giant = 0;
};
int32_t diagonal_shape(const Context &c, int64_t rows, int64_t cols, uint32_t baby, uint32_t giant, DiagonalShape &s) {
    int32_t rc = check_dimensions(c, rows, cols, s.dimension);
    if (rc) return rc;
    s.baby = (int32_t)baby, s.giant = (int32_t)giant;
    if ((int64_t)baby != s.baby || (int64_t)giant != s.giant) s.baby = s.giant = -1;
    if ((rc = check_steps(c, s.dimension, s.baby, s.giant))) return rc;
    if (!c.simd) return fail(HECUDA_ERR_UNSUPPORTED, "simdEncodingNotSupported");
    s.results = (rows + c.n - 1) / c.n;
    s.count = s.dimension * s.results;
    s.slots = s.results * s.giant * s.baby;
    return HECUDA_OK;
}

// plaintext index resultCount * (j + babyStep * g) + r  ->  slot (r, g, j), as hecuda_pnns_matrix_create places them
std::vector<long long> file_slots(const DiagonalShape &s) {
    std::vector<long long> slot((size_t)s.count);
    for (int64_t p = 0; p < s.count; ++p) {
        const int64_t r = p % s.results, d = p / s.results;
        slot[(size_t)p] = (r * s.giant + d / s.baby) * s.baby + d % s.baby;
    }
    return slot;
}

// The chunks of every matrix, in file order: (matrix, chunk of its plaintexts), and the largest chunk's bytes
struct MatrixChunk {
    int matrix;
    dbio::Chunk chunk;
};
std::vector<MatrixChunk> plan_matrix_chunks(const std::vector<std::vector<long long>> &tags, long long &widest) {
    std::vector<MatrixChunk> plan;
    widest = 1;
    for (size_t k = 0; k < tags.size(); ++k)
        for (const dbio::Chunk &ch : dbio::plan_chunks(tags[k], 0, (long long)tags[k].size() - 1, kSlabBytes)) {
            plan.push_back({(int)k, ch});
            widest = std::max(widest, tags[k][(size_t)(ch.first + ch.count)] - tags[k][(size_t)ch.first]);
        }
    return plan;
}

// Device copies of each matrix's framing offsets and slot map
struct DeviceMaps {
    std::vector<long long *> tag, slot;
    ~DeviceMaps() {
        for (long long *p : tag) cudaFree(p);
        for (long long *p : slot) cudaFree(p);
    }
    cudaError_t add(const std::vector<long long> &t, const std::vector<long long> &s) {
        tag.push_back(nullptr);
        slot.push_back(nullptr);
        cudaError_t e = cudaMalloc(&tag.back(), t.size() * sizeof(long long));
        if (e == cudaSuccess) e = upload(tag.back(), t.data(), t.size() * sizeof(long long));
        if (e == cudaSuccess) e = cudaMalloc(&slot.back(), std::max<size_t>(s.size(), 1) * sizeof(long long));
        if (e == cudaSuccess && !s.empty()) e = upload(slot.back(), s.data(), s.size() * sizeof(long long));
        return e;
    }
};

// The checks shared by the byte count and the serialization, and where everything goes.  Launches nothing.
int32_t serialization_placement(const hecuda_pnns_matrix *const *ms, int32_t count, const uint64_t *ids, int64_t id_count,
                                const uint8_t *metadata, const uint64_t *metadata_offsets, int64_t metadata_count,
                                const hecuda_pnns_server_config *cfg, pnnsio::Placement &pl, std::vector<DiagonalShape> &shapes,
                                std::vector<CodecConsts> &cc) {
    if (!ms || count < 1 || !cfg) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / no matrices");
    if (id_count < 0 || metadata_count < 0 || (id_count && !ids) || (metadata_count && !metadata_offsets))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null or negative entry buffers");
    for (int64_t k = 0; k < metadata_count; ++k)
        if (metadata_offsets[k + 1] < metadata_offsets[k])
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "metadata offsets must not decrease");
    if (metadata_count && metadata_offsets[metadata_count] > metadata_offsets[0] && !metadata)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null metadata");
    pnnsio::Error e;
    if (!pnnsio::check_config(*cfg, true, e)) return io_fail(e);
    if (cfg->database_packing != pnnsio::kDiagonal)
        return fail(HECUDA_ERR_UNSUPPORTED, "databasePacking: only .diagonal matrices are resident here");
    std::vector<const hecuda_context *> ctxs((size_t)count);
    for (int32_t k = 0; k < count; ++k) {
        if (!ms[k]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null matrix");
        ctxs[(size_t)k] = ms[k]->owner;
    }
    int32_t rc = validate_contexts(ctxs.data(), count, *cfg);
    if (rc) return rc;
    std::vector<pnnsio::MatrixShape> placed;
    for (int32_t k = 0; k < count; ++k) {
        const hecuda_pnns_matrix *m = ms[k];
        const Context &c = *m->owner->ctx;
        if (m->row_count != ms[0]->row_count || m->column_count != ms[0]->column_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "the matrices differ in shape");
        if ((uint32_t)m->baby != cfg->database_baby_step || (uint32_t)m->giant != cfg->database_giant_step)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongMatrixPacking: the config's babyStep / giantStep are not the matrix's");
        shapes.emplace_back();
        if ((rc = diagonal_shape(c, m->row_count, m->column_count, (uint32_t)m->baby, (uint32_t)m->giant, shapes.back()))) return rc;
        cc.emplace_back();
        std::string err;
        if (!codec_consts(c, c.map_q(c.L), 0, cc.back(), err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
        placed.push_back({m->row_count, m->column_count, shapes.back().count, serialized_poly_bytes(cc.back())});
    }
    pl = pnnsio::place_database(placed, ids, id_count, metadata, metadata_offsets, metadata_count, *cfg);
    return HECUDA_OK;
}

// A standalone config message: its bytes into `out`, or only their count with out = NULL
int32_t write_message(const pnnsio::Bytes &bytes, uint8_t *out, uint64_t capacity, uint64_t *written) {
    if (!out) {
        *written = bytes.size();
        return HECUDA_OK;
    }
    if (capacity < bytes.size())
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below the serialized size " +
                                                     std::to_string(bytes.size()));
    memcpy(out, bytes.data(), bytes.size());
    *written = bytes.size();
    return HECUDA_OK;
}

long long clamp_size(uint64_t byte_count) { return (long long)std::min<uint64_t>(byte_count, INT64_MAX); }

}  // namespace

extern "C" {

int32_t hecuda_pnns_server_config_parse(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *out) {
    if (!out || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    hecuda_pnns_server_config c{};
    pnnsio::Error e;
    if (!pnnsio::parse_server_config(bytes, 0, clamp_size(byte_count), c, e)) return io_fail(e);
    *out = c;
    return HECUDA_OK;
}

int32_t hecuda_pnns_client_config_parse(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *out) {
    if (!out || (!bytes && byte_count)) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    hecuda_pnns_server_config c{};
    pnnsio::Error e;
    if (!pnnsio::parse_client_config(bytes, 0, clamp_size(byte_count), c, e)) return io_fail(e);
    *out = c;
    return HECUDA_OK;
}

int32_t hecuda_pnns_server_config_serialize(const hecuda_pnns_server_config *config, uint8_t *out, uint64_t capacity,
                                            uint64_t *written) {
    if (!config || !written) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *written = 0;
    pnnsio::Error e;
    if (!pnnsio::check_config(*config, true, e)) return io_fail(e);
    return write_message(pnnsio::encode_server_config(*config), out, capacity, written);
}

int32_t hecuda_pnns_client_config_serialize(const hecuda_pnns_server_config *config, uint8_t *out, uint64_t capacity,
                                            uint64_t *written) {
    if (!config || !written) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *written = 0;
    pnnsio::Error e;
    if (!pnnsio::check_config(*config, false, e)) return io_fail(e);
    return write_message(pnnsio::encode_client_config(*config), out, capacity, written);
}

int32_t hecuda_pnns_database_describe(const uint8_t *bytes, uint64_t byte_count, hecuda_pnns_server_config *config,
                                      int32_t *matrix_count, int64_t *row_count, int64_t *column_count,
                                      int64_t *entry_id_count, int64_t *metadata_count, uint64_t *metadata_bytes) {
    if (!config || !matrix_count || !row_count || !column_count || !entry_id_count || !metadata_count || !metadata_bytes ||
        (!bytes && byte_count))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsio::Database db;
    pnnsio::Error e;
    if (!pnnsio::walk_database(bytes, clamp_size(byte_count), db, e)) return io_fail(e);
    for (const pnnsio::Matrix &m : db.matrices)
        if (m.rows != db.matrices[0].rows || m.cols != db.matrices[0].cols)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "the plaintext matrices differ in num_rows / num_columns");
    *config = db.config;
    *matrix_count = (int32_t)db.matrices.size();
    *row_count = db.matrices.empty() ? 0 : db.matrices[0].rows;
    *column_count = db.matrices.empty() ? 0 : db.matrices[0].cols;
    *entry_id_count = (int64_t)db.entry_ids.size();
    *metadata_count = (int64_t)db.metadata_bytes.size();
    uint64_t total = 0;
    for (long long b : db.metadata_bytes) total += (uint64_t)b;
    *metadata_bytes = total;
    return HECUDA_OK;
}

int32_t hecuda_pnns_database_entries(const uint8_t *bytes, uint64_t byte_count, uint64_t *entry_ids, int64_t id_capacity,
                                     uint8_t *metadata, uint64_t metadata_capacity, uint64_t *metadata_offsets,
                                     int64_t offsets_capacity) {
    if (!bytes && byte_count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsio::Database db;
    pnnsio::Error e;
    if (!pnnsio::walk_database(bytes, clamp_size(byte_count), db, e)) return io_fail(e);
    if (entry_ids) {
        if (id_capacity < (int64_t)db.entry_ids.size()) return fail(HECUDA_ERR_INVALID_ARGUMENT, "id_capacity below the entry count");
        std::copy(db.entry_ids.begin(), db.entry_ids.end(), entry_ids);
    }
    uint64_t total = 0;
    for (long long b : db.metadata_bytes) total += (uint64_t)b;
    if (metadata_offsets && offsets_capacity < (int64_t)db.metadata_bytes.size() + 1)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "offsets_capacity below the metadata count + 1");
    if (metadata && metadata_capacity < total) return fail(HECUDA_ERR_INVALID_ARGUMENT, "metadata_capacity below the metadata bytes");
    uint64_t at = 0;
    for (size_t k = 0; k < db.metadata_bytes.size(); ++k) {
        if (metadata_offsets) metadata_offsets[k] = at;
        if (metadata) memcpy(metadata + at, bytes + db.metadata_at[k], (size_t)db.metadata_bytes[k]);
        at += (uint64_t)db.metadata_bytes[k];
    }
    if (metadata_offsets) metadata_offsets[db.metadata_bytes.size()] = at;
    return HECUDA_OK;
}

int32_t hecuda_pnns_matrices_create_serialized(const hecuda_context *const *ctxs, int32_t count, const uint8_t *bytes,
                                               uint64_t byte_count, hecuda_pnns_matrix **out) {
    if (!out || !ctxs || count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument or no context");
    for (int32_t k = 0; k < count; ++k) out[k] = nullptr;
    if (!bytes && byte_count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    // every check before anything is allocated
    pnnsio::Database db;
    pnnsio::Error e;
    if (!pnnsio::walk_database(bytes, clamp_size(byte_count), db, e)) return io_fail(e);
    int32_t rc = validate_contexts(ctxs, count, db.config);
    if (rc) return rc;
    if ((int32_t)db.matrices.size() != count)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidDatabase: " + std::to_string(db.matrices.size()) +
                                                     " plaintext matrices for " + std::to_string(count) + " plaintext moduli");
    if (db.config.database_packing != pnnsio::kDiagonal)
        return fail(HECUDA_ERR_UNSUPPORTED, "databasePacking: only .diagonal matrices are resident here");
    std::vector<DiagonalShape> shapes((size_t)count);
    std::vector<CodecConsts> cc((size_t)count);
    std::vector<std::vector<long long>> tags((size_t)count);
    for (int32_t k = 0; k < count; ++k) {
        const pnnsio::Matrix &m = db.matrices[(size_t)k];
        const Context &c = *ctxs[k]->ctx;
        const std::string which = "matrix " + std::to_string(k);
        if (m.packing != pnnsio::kDiagonal)
            return fail(HECUDA_ERR_UNSUPPORTED, which + ": only .diagonal matrices are resident here");
        DiagonalShape &s = shapes[(size_t)k];
        if ((rc = diagonal_shape(c, m.rows, m.cols, m.bsgs[1], m.bsgs[2], s))) return rc;
        if ((int64_t)m.poly_at.size() != s.count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "wrongPlaintextCount(got: " + std::to_string(m.poly_at.size()) +
                                                         ", expected: " + std::to_string(s.count) + ") in " + which);
        std::string err;
        if (!codec_consts(c, c.map_q(c.L), 0, cc[(size_t)k], err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
        const long long poly_bytes = serialized_poly_bytes(cc[(size_t)k]);
        for (size_t p = 0; p < m.poly_bytes.size(); ++p)
            if (m.poly_bytes[p] != poly_bytes)
                return fail(HECUDA_ERR_INVALID_ARGUMENT, "corruptedData(" + which + ", plaintext " + std::to_string(p) + ": " +
                                                             std::to_string(m.poly_bytes[p]) + " bytes of poly, expected " +
                                                             std::to_string(poly_bytes) + " for " + std::to_string(c.L) + " rows)");
        // the rows' own offsets (frame 0); the last plaintext ends its matrix's stream
        tags[(size_t)k] = m.poly_at;
        tags[(size_t)k].push_back(m.poly_at.back() + poly_bytes);
    }
    long long widest = 0;
    const std::vector<MatrixChunk> plan = plan_matrix_chunks(tags, widest);
    long long last = 0;
    for (const std::vector<long long> &t : tags) last = std::max(last, t.back());
    const bool pinned = host_pinned(bytes, (size_t)last);

    DbStaging st(ctxs[0]);
    if (!st.g0.w || !st.g1.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    std::vector<hecuda_pnns_matrix *> ms;
    DeviceMaps maps;
    unsigned long long *d_bad = nullptr;
    std::vector<unsigned long long> bad((size_t)count, ~0ull);
    cudaError_t err = cudaSuccess;
    for (int32_t k = 0; k < count && err == cudaSuccess; ++k) {
        const Context &c = *ctxs[k]->ctx;
        const DiagonalShape &s = shapes[(size_t)k];
        hecuda_pnns_matrix *m = new (std::nothrow) hecuda_pnns_matrix();
        if (!m) {
            err = cudaErrorMemoryAllocation;
            break;
        }
        ms.push_back(m);
        m->owner = ctxs[k];
        m->row_count = db.matrices[(size_t)k].rows;
        m->column_count = db.matrices[(size_t)k].cols;
        m->result_count = s.results;
        m->baby = s.baby;
        m->giant = s.giant;
        m->dimension = (int)s.dimension;
        // slots past the padded dimension are absent: zero rows, flag 0
        std::vector<unsigned char> present((size_t)s.slots);
        for (int64_t slot = 0; slot < s.slots; ++slot) present[(size_t)slot] = slot % ((int64_t)s.giant * s.baby) < s.dimension;
        const size_t words = (size_t)c.L * c.n * s.slots;
        err = cudaMalloc(&m->d_plain, words * sizeof(u64));
        if (err == cudaSuccess) err = fill(m->d_plain, 0, words * sizeof(u64));
        if (err == cudaSuccess) err = cudaMalloc(&m->d_present, (size_t)s.slots);
        if (err == cudaSuccess) err = upload(m->d_present, present.data(), (size_t)s.slots);
        if (err == cudaSuccess) err = maps.add(tags[(size_t)k], file_slots(s));
    }
    if (err == cudaSuccess) err = cudaMalloc(&d_bad, (size_t)count * sizeof(unsigned long long));
    if (err == cudaSuccess) err = fill(d_bad, 0xff, (size_t)count * sizeof(unsigned long long));
    if (err == cudaSuccess) err = st.init((size_t)widest, !pinned);
    for (size_t k = 0; k < plan.size() && err == cudaSuccess; ++k) {
        const int b = (int)(k & 1), mi = plan[k].matrix;
        const dbio::Chunk &ch = plan[k].chunk;
        const std::vector<long long> &tag = tags[(size_t)mi];
        const long long base = tag[(size_t)ch.first], size = tag[(size_t)(ch.first + ch.count)] - base;
        const unsigned char *src = bytes + base;
        if (!pinned) {  // the pinned buffer is free once the copy two chunks back has finished
            if (k >= 2) err = cudaEventSynchronize(st.copied[b]);
            if (err != cudaSuccess) break;
            memcpy(st.host[b], src, (size_t)size);
            src = st.host[b];
        }
        err = cudaMemcpyAsync(st.dev[b], src, (size_t)size, cudaMemcpyHostToDevice, st.stream[b]);
        if (err == cudaSuccess && !pinned) err = cudaEventRecord(st.copied[b], st.stream[b]);
        PolyLayout at;
        at.tag = maps.tag[(size_t)mi];
        at.base = base;
        at.first = ch.first;
        at.bad = d_bad + mi;
        at.slot = maps.slot[(size_t)mi];
        at.frame = 0;
        if (err == cudaSuccess)
            err = launch_poly_load(*ctxs[mi]->ctx, cc[(size_t)mi], 0, st.dev[b], ms[(size_t)mi]->d_plain, ch.count, st.stream[b], at);
    }
    for (int b = 0; b < 2; ++b) {
        const cudaError_t e2 = cudaStreamSynchronize(st.stream[b]);
        if (err == cudaSuccess) err = e2;
    }
    if (err == cudaSuccess) err = cudaMemcpy(bad.data(), d_bad, (size_t)count * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    cudaFree(d_bad);
    const auto first_bad = std::find_if(bad.begin(), bad.end(), [](unsigned long long v) { return v != ~0ull; });
    if (err == cudaSuccess && first_bad == bad.end()) {
        for (int32_t k = 0; k < count; ++k) out[k] = ms[(size_t)k];
        return HECUDA_OK;
    }
    for (hecuda_pnns_matrix *m : ms) hecuda_pnns_matrix_destroy(m);
    if (err != cudaSuccess) return cuda_fail(err, "pnns matrices from serialized bytes");
    const int mi = (int)(first_bad - bad.begin());
    const int L = ctxs[mi]->ctx->L;
    const int row = (int)(*first_bad % (unsigned long long)L);
    return fail(HECUDA_ERR_INVALID_ARGUMENT, "corruptedData(matrix " + std::to_string(mi) + ", plaintext " +
                                                 std::to_string(*first_bad / (unsigned long long)L) + ", row " +
                                                 std::to_string(row) + ": a residue is not below q_" + std::to_string(row) +
                                                 " = " + std::to_string(cc[(size_t)mi].modulus[row]) + ")");
}

int32_t hecuda_pnns_database_serialized_byte_count(const hecuda_pnns_matrix *const *matrices, int32_t count,
                                                   const uint64_t *entry_ids, int64_t entry_id_count,
                                                   const uint8_t *metadata, const uint64_t *metadata_offsets,
                                                   int64_t metadata_count, const hecuda_pnns_server_config *config,
                                                   uint64_t *bytes) {
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    pnnsio::Placement pl;
    std::vector<DiagonalShape> shapes;
    std::vector<CodecConsts> cc;
    int32_t rc = serialization_placement(matrices, count, entry_ids, entry_id_count, metadata, metadata_offsets,
                                         metadata_count, config, pl, shapes, cc);
    if (rc) return rc;
    *bytes = (uint64_t)pl.size;
    return HECUDA_OK;
}

int32_t hecuda_pnns_database_serialize(const hecuda_pnns_matrix *const *matrices, int32_t count, const uint64_t *entry_ids,
                                       int64_t entry_id_count, const uint8_t *metadata, const uint64_t *metadata_offsets,
                                       int64_t metadata_count, const hecuda_pnns_server_config *config, uint8_t *out,
                                       uint64_t capacity, uint64_t *written) {
    if (!out || !written) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *written = 0;
    pnnsio::Placement pl;
    std::vector<DiagonalShape> shapes;
    std::vector<CodecConsts> cc;
    int32_t rc = serialization_placement(matrices, count, entry_ids, entry_id_count, metadata, metadata_offsets,
                                         metadata_count, config, pl, shapes, cc);
    if (rc) return rc;
    if (capacity < (uint64_t)pl.size)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below the serialized size " +
                                                     std::to_string(pl.size));
    // the bytes around the plaintexts come from the host
    for (const pnnsio::MatrixPlacement &mp : pl.matrices) {
        memcpy(out + mp.head_at, mp.head.data(), mp.head.size());
        memcpy(out + mp.tag.back(), mp.tail.data(), mp.tail.size());
    }
    memcpy(out + pl.rest_at, pl.rest.data(), pl.rest.size());
    std::vector<std::vector<long long>> tags;
    for (const pnnsio::MatrixPlacement &mp : pl.matrices) tags.push_back(mp.tag);
    long long widest = 0;
    const std::vector<MatrixChunk> plan = plan_matrix_chunks(tags, widest);
    const bool pinned = host_pinned(out, (size_t)pl.size);
    DbStaging st(matrices[0]->owner);
    if (!st.g0.w || !st.g1.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    DeviceMaps maps;
    cudaError_t e = cudaSuccess;
    for (int32_t k = 0; k < count && e == cudaSuccess; ++k) e = maps.add(tags[(size_t)k], file_slots(shapes[(size_t)k]));
    if (e == cudaSuccess) e = st.init((size_t)widest, !pinned);
    auto range = [&](size_t k, long long &base) {
        const dbio::Chunk &ch = plan[k].chunk;
        const std::vector<long long> &tag = tags[(size_t)plan[k].matrix];
        base = tag[(size_t)ch.first];
        return tag[(size_t)(ch.first + ch.count)] - base;
    };
    // a pageable `out`: chunk k's pinned bytes are copied out once chunk k + 1 is enqueued
    auto drain = [&](size_t k) {
        long long base = 0;
        const long long size = range(k, base);
        cudaError_t e2 = cudaEventSynchronize(st.copied[k & 1]);
        if (e2 == cudaSuccess) memcpy(out + base, st.host[k & 1], (size_t)size);
        return e2;
    };
    for (size_t k = 0; k < plan.size() && e == cudaSuccess; ++k) {
        const int b = (int)(k & 1), mi = plan[k].matrix;
        const pnnsio::MatrixPlacement &mp = pl.matrices[(size_t)mi];
        long long base = 0;
        const long long size = range(k, base);
        PolyLayout at;
        at.tag = maps.tag[(size_t)mi];
        at.base = base;
        at.first = plan[k].chunk.first;
        at.slot = maps.slot[(size_t)mi];
        at.frame = (int)mp.frame.size();
        std::copy(mp.frame.begin(), mp.frame.end(), at.frame_bytes);
        e = launch_poly_serialize(*matrices[mi]->owner->ctx, cc[(size_t)mi], 0, (const u64 *)matrices[mi]->d_plain, st.dev[b],
                                  plan[k].chunk.count, st.stream[b], at);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(pinned ? out + base : st.host[b], st.dev[b], (size_t)size, cudaMemcpyDeviceToHost, st.stream[b]);
        if (e == cudaSuccess && !pinned) e = cudaEventRecord(st.copied[b], st.stream[b]);
        if (e == cudaSuccess && !pinned && k >= 1) e = drain(k - 1);
    }
    if (e == cudaSuccess && !pinned && !plan.empty()) e = drain(plan.size() - 1);
    for (int b = 0; b < 2; ++b) {
        const cudaError_t e2 = cudaStreamSynchronize(st.stream[b]);
        if (e == cudaSuccess) e = e2;
    }
    if (e != cudaSuccess) return cuda_fail(e, "pnns database serialize");
    *written = (uint64_t)pl.size;
    return HECUDA_OK;
}

}  // extern "C"
