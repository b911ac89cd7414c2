// pir.cu -- MulPir index-PIR server pipeline on one device (SURVEY.md 8f rank 3).
//
//   PirUtil.expand / expandCiphertext / expandCiphertextForOneStep   IndexPir/PirUtil.swift:204-355
//   PirUtil.computeResponse / computeResponseForOneChunk            IndexPir/PirUtil.swift:408-568
//   MulPirServer.process output layout (column-major first dimension) IndexPir/MulPir.swift:433-556
//   modSwitchDownToSingle                                            HeScheme.swift:1481-1485
//
// The reference walks the expansion tree recursively and fans the database columns out to Swift tasks.  Here the tree
// is processed level by level: all nodes of a level go through ONE batched applyGalois (Galois permutation + hybrid
// key switch) and ONE combine kernel that forms  p0 = c1 + ct  and  p1 = x^(-2^(logStep-1)) (ct - c1)  and writes
// leaves (doubled where the reference adds the ciphertext to itself) straight to their final, interleaved position.
// The first dimension is one streaming pass over the device-resident plaintext database
// (inner_product_plain_kernel), further dimensions are lazy ct x ct inner products + relinearization.
// One pipeline (respond_group) answers every call: a group of up to HECUDA_MULPIR_CLIENT_GROUP clients goes through
// each stage in one pass, each client with its own keys, and a group of one runs the single-client kernels.
// Everything is enqueued on one stream; concurrent calls run on different streams from different host threads.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include <set>

#include "capi_internal.hpp"
#include "database_io.hpp"
#include "pir_proto.hpp"
#include "proto_respond.hpp"
#include "wire_codec.hpp"

using namespace hecuda;
using namespace hecuda::api;

struct hecuda_pir_database {
    const hecuda_context *owner = nullptr;
    u64 *d_plain = nullptr;              // count x L x N, Eval format; all-zero rows where present == 0
    u32 *d_plain32 = nullptr;            // the same rows as uint32 instead, when every ciphertext modulus is below 2^31
    unsigned char *d_present = nullptr;  // count; null = all present
    int64_t count = 0;
};

namespace {

// one node of an expansion level: where its two children go
struct ExpandStep {
    int dst0, dst1;
    unsigned flags;  // 1: p0 is a leaf (goes to `out`), 2: p0 doubled, 4: p1 is a leaf, 8: p1 doubled
};

// expandCiphertextForOneStep after the Galois step (PirUtil.swift:230-235) for every node of a level:
//   p0 = c1 + ct,  p1 = multiplyPowerOfX(ct - c1, -2^(logStep-1))   [gather form of PolyRq.swift:398-422]
// Item item0 + blockIdx.z is node (item % nodes) of client (item / nodes); a client's children go `next_cts`
// ciphertexts into `next` and its leaves `out_cts` ciphertexts into `out` after the previous client's.
__global__ void __launch_bounds__(256) expand_combine_kernel(const u64 *__restrict__ cur, const u64 *__restrict__ c1,
                                                            u64 *__restrict__ next, u64 *__restrict__ out,
                                                            const ExpandStep *__restrict__ steps,
                                                            const __grid_constant__ RowModuli c, int logn, unsigned s,
                                                            int64_t item0, int nodes, int64_t next_cts, int64_t out_cts) {
    const int n = 1 << logn;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int pr = blockIdx.y;  // poly * rows + row
    const u64 p = c.p[pr % c.rows];
    const int64_t ct_words = (int64_t)2 * c.rows * n;
    const int64_t item = item0 + blockIdx.z, client = item / nodes;
    const int64_t base = item * ct_words + (int64_t)pr * n;
    const ExpandStep st = steps[item - client * nodes];
    next += client * next_cts * ct_words;
    out += client * out_cts * ct_words;
    u64 sum = add_mod(cur[base + e], c1[base + e], p);
    const unsigned raw = ((unsigned)e - s) & (2u * n - 1u);
    const unsigned src = raw & (n - 1u);
    const u64 a = cur[base + src], b = c1[base + src];
    u64 d = a >= b ? a - b : a + p - b;
    if (raw >= (unsigned)n && d != 0) d = p - d;
    if (st.flags & 2u) sum = add_mod(sum, sum, p);
    if (st.flags & 8u) d = add_mod(d, d, p);
    ((st.flags & 1u) ? out : next)[(int64_t)st.dst0 * ct_words + (int64_t)pr * n + e] = sum;
    ((st.flags & 4u) ? out : next)[(int64_t)st.dst1 * ct_words + (int64_t)pr * n + e] = d;
}

int ceil_log2(int64_t x) {
    int k = 0;
    while (((int64_t)1 << k) < x) ++k;
    return k;
}
int floor_log2(int64_t x) {
    int k = 0;
    while (((int64_t)2 << k) <= x) ++k;
    return k;
}

// ---- host-side plan of the expansion tree -------------------------------------------------------------------
struct PlanNode {
    int64_t count;
    int height;                      // expectedHeight of its root
    std::vector<int64_t> positions;  // final output positions of this node's outputs, in order
};
struct PlanLevel {
    int log_step;
    int64_t nodes;        // all of them active (count > 1)
    size_t step_offset;   // into ExpandPlan::steps
};
struct ExpandPlan {
    std::vector<PlanLevel> levels;
    std::vector<ExpandStep> steps;
    std::vector<std::pair<int64_t, int64_t>> root_leaves;  // (input ciphertext, output position): copied as is
    int64_t active_roots = 0, max_nodes = 0;
};

ExpandPlan build_expand_plan(int64_t n, int64_t ct_count, int64_t output_count) {
    ExpandPlan plan;
    std::vector<PlanNode> cur;
    int64_t remaining = output_count, offset = 0;
    for (int64_t i = 0; i < ct_count; ++i) {  // PirUtil.expand: lengths (PirUtil.swift:328-333)
        const int64_t count = std::min(remaining, n);
        remaining -= count;
        if (count == 1) {  // expandCiphertext with outputCount == 1 at logStep 1 > expectedHeight 0: returned unchanged
            plan.root_leaves.push_back({i, offset});
        } else if (count > 1) {
            PlanNode node{count, ceil_log2(count), {}};
            node.positions.resize(count);
            for (int64_t j = 0; j < count; ++j) node.positions[j] = offset + j;
            cur.push_back(std::move(node));
        }
        offset += count;
    }
    plan.active_roots = (int64_t)cur.size();
    int log_step = 1;
    while (!cur.empty()) {
        PlanLevel level{log_step, (int64_t)cur.size(), plan.steps.size()};
        plan.max_nodes = std::max<int64_t>(plan.max_nodes, level.nodes);
        std::vector<PlanNode> next;
        for (const PlanNode &node : cur) {
            const int64_t second = node.count >> 1, first = node.count - second;
            PlanNode child[2] = {{first, node.height, {}}, {second, node.height, {}}};
            for (int64_t j = 0; j < second; ++j) {  // zip(firstHalf.prefix(second), secondHalf) interleaved (:302)
                child[0].positions.push_back(node.positions[2 * j]);
                child[1].positions.push_back(node.positions[2 * j + 1]);
            }
            for (int64_t j = 2 * second; j < node.count; ++j) child[0].positions.push_back(node.positions[j]);
            ExpandStep st{0, 0, 0u};
            for (int k = 0; k < 2; ++k) {
                int dst;
                if (child[k].count == 1) {
                    dst = (int)child[k].positions[0];
                    st.flags |= (k ? 4u : 1u);
                    if (log_step + 1 <= node.height) st.flags |= (k ? 8u : 2u);  // output += ciphertext (:260-264)
                } else {
                    dst = (int)next.size();
                    next.push_back(std::move(child[k]));
                }
                (k ? st.dst1 : st.dst0) = dst;
            }
            plan.steps.push_back(st);
        }
        plan.levels.push_back(level);
        cur.swap(next);
        ++log_step;
    }
    return plan;
}

// the largest configured Galois element <= target and how many times to apply it (PirUtil.swift:213-228)
int32_t pick_galois(const hecuda_evk *k, int64_t n, int log_step, unsigned *element, int *times, const u64 **key) {
    const int logn = floor_log2(n);
    const unsigned target = (1u << (logn - log_step + 1)) + 1u;
    hecuda_evk *km = const_cast<hecuda_evk *>(k);
    std::lock_guard<std::mutex> g(km->mu);
    unsigned best = 0;
    const u64 *best_key = nullptr;
    for (const auto &kv : km->galois)
        if (kv.first <= target && kv.first > best) {
            best = kv.first;
            best_key = kv.second;
        }
    if (!best) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey");
    const int count = 1 << (floor_log2(target - 1) - floor_log2(best - 1));
    unsigned long long cur = 1;
    for (int i = 0; i < count; ++i) cur = cur * best % (unsigned long long)(2 * n);
    if (cur != target) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey: configured elements cannot reach " + std::to_string(target));
    *element = best;
    *times = count;
    *key = best_key;
    return HECUDA_OK;
}

// The Galois element, repeat count and key that every expansion level of `plan` applies, for clients
// first_client .. first_client + clients - 1 (keys[j] belongs to client first_client + j).  All clients must resolve
// to the same element at every level.  first_client < 0: one client answered alone, whose errors name no client.
struct LevelKeys {
    unsigned element = 0;
    int times = 0;
    std::vector<const u64 *> key;  // [j]
};
int32_t resolve_level_keys(const hecuda_evk *const *keys, int clients, int first_client, int64_t n, const ExpandPlan &plan,
                           std::vector<LevelKeys> &out) {
    out.assign(plan.levels.size(), LevelKeys{});
    const int first = std::max(first_client, 0);
    for (size_t li = 0; li < plan.levels.size(); ++li) {
        LevelKeys &lk = out[li];
        lk.key.resize((size_t)clients);
        for (int j = 0; j < clients; ++j) {
            unsigned element = 0;
            int times = 0;
            const std::string who = "client " + std::to_string(first + j);
            int32_t rc32 = pick_galois(keys[j], n, plan.levels[li].log_step, &element, &times, &lk.key[j]);
            if (rc32) return first_client < 0 ? rc32 : fail(rc32, who + ": " + last_error_cstr());
            if (j > 0 && (element != lk.element || times != lk.times))
                return fail(HECUDA_ERR_INVALID_ARGUMENT,
                            who + ": its Galois keys apply element " + std::to_string(element) + " at expansion level " +
                                std::to_string(plan.levels[li].log_step) + ", client " + std::to_string(first) +
                                "'s apply " + std::to_string(lk.element) + "; answer it with hecuda_mulpir_compute_response");
            lk.element = element;
            lk.times = times;
        }
    }
    return HECUDA_OK;
}

// The expansion plan of a query shape on the device, uploaded the first time the context sees the shape, so that
// later calls enqueue without waiting for a copy.  The upload runs outside the context's lock; when two threads race
// on a new shape, the second copy is dropped.
int32_t expand_steps_on_device(const hecuda_context *hc, int64_t n, int64_t ct_count, int64_t output_count, const ExpandStep **out) {
    hecuda_context *h = const_cast<hecuda_context *>(hc);
    const std::pair<int64_t, int64_t> shape{ct_count, output_count};
    {
        std::lock_guard<std::mutex> lock(h->mu);
        auto it = h->expand_steps.find(shape);
        if (it != h->expand_steps.end()) {
            *out = (const ExpandStep *)it->second;
            return HECUDA_OK;
        }
    }
    const ExpandPlan plan = build_expand_plan(n, ct_count, output_count);
    void *d = nullptr;
    cudaError_t e = cudaMalloc(&d, std::max<size_t>(plan.steps.size(), 1) * sizeof(ExpandStep));
    if (e == cudaSuccess && !plan.steps.empty()) e = upload(d, plan.steps.data(), plan.steps.size() * sizeof(ExpandStep));
    if (e != cudaSuccess) {
        if (d) cudaFree(d);
        return cuda_fail(e, "expansion plan upload");
    }
    std::lock_guard<std::mutex> lock(h->mu);
    auto ins = h->expand_steps.insert({shape, d});
    if (!ins.second) cudaFree(d);  // another thread uploaded the same plan first; nothing has used this copy
    *out = (const ExpandStep *)ins.first->second;
    return HECUDA_OK;
}

// PirUtil.expand on device buffers for `clients` queries of the same shape: client j's ct_count canonical (Coeff)
// ciphertexts of L rows at d_in + j * ct_count ciphertexts, its output_count outputs at d_out + j * output_count,
// expanded with keys[j].  Every stage is one pass over all clients.
// first_client: the call-wide index of keys[0] for error messages (resolve_level_keys)
int32_t expand_device(const hecuda_context *h, const hecuda_evk *const *keys, int clients, const u64 *d_in, int64_t ct_count,
                      int64_t output_count, u64 *d_out, cudaStream_t s, int first_client = -1) {
    const Context &c = *h->ctx;
    const int l = c.L;
    const int64_t n = c.n;
    const size_t ct_words = (size_t)2 * l * n;
    const ExpandPlan plan = build_expand_plan(n, ct_count, output_count);
    // resolve every level's Galois key for every client before anything is enqueued
    std::vector<LevelKeys> level_keys;
    int32_t rc_keys = resolve_level_keys(keys, clients, first_client, n, plan, level_keys);
    if (rc_keys) return rc_keys;
    if (clients > kKeyTableSize) return fail(HECUDA_ERR_UNSUPPORTED, "expand: more clients than one key table holds");
    const ExpandStep *d_steps = nullptr;
    if ((rc_keys = expand_steps_on_device(h, n, ct_count, output_count, &d_steps))) return rc_keys;
    std::vector<KsKeyTable> tables(plan.levels.size(), KsKeyTable{});
    for (size_t li = 0; li < plan.levels.size(); ++li) {
        tables[li].items_per_client = plan.levels[li].nodes;
        for (int j = 0; j < clients && j < kKeyTableSize; ++j) tables[li].key[j] = level_keys[li].key[j];
    }
    const size_t in_pitch = ct_words * ct_count * sizeof(u64), out_pitch = ct_words * output_count * sizeof(u64);
    for (const auto &leaf : plan.root_leaves)
        CK(cudaMemcpy2DAsync(d_out + ct_words * leaf.second, out_pitch, d_in + ct_words * leaf.first, in_pitch,
                             ct_words * sizeof(u64), (size_t)clients, cudaMemcpyDeviceToDevice, s));
    if (plan.levels.empty()) return HECUDA_OK;
    StreamBuffers tmp(s);
    u64 *level_buf[2] = {nullptr, nullptr}, *c1_buf[2] = {nullptr, nullptr}, *scratch = nullptr;
    // items per applyGalois pass: grows with the number of clients, so the launch count does not
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, plan.max_nodes)) * clients;
    const size_t level_words = ct_words * plan.max_nodes * clients;
    CK(tmp.alloc(&level_buf[0], level_words));
    CK(tmp.alloc(&level_buf[1], level_words));
    CK(tmp.alloc(&c1_buf[0], level_words));
    CK(tmp.alloc(&c1_buf[1], level_words));
    CK(tmp.alloc(&scratch, galois_scratch_words(c, l) * (size_t)chunk));
    const RowModuli rc = row_moduli(c, c.map_q(l));
    const int threads = coeff_threads(n);
    // the active roots are a prefix of each input (only the last one can be a single output); a level's nodes must be
    // contiguous over all clients, so several clients' roots are gathered when a single-output root sits between them
    const u64 *cur = d_in;
    if (clients > 1 && plan.active_roots != ct_count) {
        CK(cudaMemcpy2DAsync(level_buf[1], ct_words * plan.active_roots * sizeof(u64), d_in, in_pitch,
                             ct_words * plan.active_roots * sizeof(u64), (size_t)clients, cudaMemcpyDeviceToDevice, s));
        cur = level_buf[1];
    }
    int flip = 0;
    for (size_t li = 0; li < plan.levels.size(); ++li) {
        const PlanLevel &level = plan.levels[li];
        const LevelKeys &lk = level_keys[li];
        KsKeyTable &table = tables[li];
        const int64_t total = level.nodes * clients;
        const u64 *c1 = cur;
        for (int t = 0; t < lk.times; ++t) {  // c1.applyGalois(element:using:) `times` times (:223-227)
            u64 *dst = c1_buf[t & 1];
            for (int64_t done = 0; done < total; done += chunk) {
                const int64_t items = std::min<int64_t>(chunk, total - done);
                table.item0 = done;
                cudaError_t e = apply_galois_chunk(c, scratch, lk.key[0], c1 + ct_words * done, l, lk.element,
                                                   dst + ct_words * done, items, s, clients > 1 ? &table : nullptr);
                if (e != cudaSuccess) return cuda_fail(e, "expand: applyGalois");
            }
            c1 = dst;
        }
        u64 *next = level_buf[flip];
        flip ^= 1;
        const int64_t next_nodes = li + 1 < plan.levels.size() ? plan.levels[li + 1].nodes : 0;
        const unsigned shift = (unsigned)(2 * n) - (1u << (level.log_step - 1));  // -2^(logStep-1) mod 2N
        const cudaError_t e = for_each_part(total, [&](int64_t done, int64_t items) {
            dim3 grid((unsigned)((n + threads - 1) / threads), (unsigned)(2 * l), (unsigned)items);
            return launch(expand_combine_kernel, grid, threads, 0, s, cur, c1, next, d_out, d_steps + level.step_offset, rc, c.logn,
                          shift, done, (int)level.nodes, next_nodes, output_count);
        });
        if (e != cudaSuccess) return cuda_fail(e, "expand: combine");
        cur = next;
    }
    return HECUDA_OK;
}

int32_t check_expand_args(const hecuda_context *h, const hecuda_evk *k, const uint64_t *cts, int64_t ct_count,
                          int64_t output_count, const void *out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (!cts || !out || ct_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidCiphertext: null buffer");
    const int64_t n = h->ctx->n;
    if (!((ct_count - 1) * n < output_count && output_count <= ct_count * n))  // preconditions, PirUtil.swift:326-327
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "expand: outputCount does not match the number of query ciphertexts");
    if (output_count > 0x7fffffff) return fail(HECUDA_ERR_UNSUPPORTED, "expand: too many outputs");
    return HECUDA_OK;
}

struct ResponseShape {
    std::vector<int64_t> dims;
    int64_t chunk_count, per_chunk, columns, expanded_query_count;
};

int32_t check_response_args(const hecuda_context *h, const hecuda_evk *k, const hecuda_pir_database *const *dbs,
                            int32_t db_count, const int32_t *dims, int32_t dim_count, int32_t chunk_count,
                            const uint64_t *query, int32_t query_ct_count, int32_t indices_count, const void *out,
                            ResponseShape &shape) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!k) return fail(HECUDA_ERR_MISSING_KEY, "missingGaloisKey");
    if (k->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: evaluation key belongs to another context");
    if (!dbs || !dims || !query || !out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (dim_count < 1 || chunk_count < 1 || indices_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid PIR parameter");
    if (!(db_count == 1 || db_count >= indices_count))  // PirError.invalidBatchSize (PirUtil.swift:498-500)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidBatchSize: queryCount " + std::to_string(indices_count) +
                                                     ", databaseCount " + std::to_string(db_count));
    shape.dims.assign(dims, dims + dim_count);
    shape.per_chunk = 1;
    shape.expanded_query_count = 0;
    for (int64_t d : shape.dims) {
        if (d < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalid PIR dimensions");
        shape.per_chunk *= d;
        shape.expanded_query_count += d;
    }
    shape.chunk_count = chunk_count;
    shape.columns = shape.per_chunk / shape.dims[0];
    if (!(shape.columns == 1 || shape.columns == shape.expanded_query_count - shape.dims[0]))  // precondition (:422)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "databaseColumnsCount must be 1 or the remaining expanded query count");
    if (dim_count > 1 && !k->loaded) return fail(HECUDA_ERR_MISSING_KEY, "missingRelinearizationKey");
    for (int32_t i = 0; i < db_count; ++i) {
        if (!dbs[i] || dbs[i]->owner != h) return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: database belongs to another context");
        if (dbs[i]->count != shape.chunk_count * shape.per_chunk)  // PirError.invalidDatabasePlaintextCount (MulPir.swift:352-358)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidDatabasePlaintextCount: " + std::to_string(dbs[i]->count) +
                                                         ", expected " + std::to_string(shape.chunk_count * shape.per_chunk));
    }
    return check_expand_args(h, k, query, query_ct_count, shape.expanded_query_count * indices_count, out);
}

// ---------------------------------------------------------------- many clients per call
static_assert(HECUDA_MULPIR_CLIENT_GROUP == kKeyTableSize, "one key-table entry per client of a group");
static_assert(HECUDA_MULPIR_CLIENT_GROUP == kScanClientTile * kScanClientTiles, "one scan launch per client group");

// Every client checked like a single call, and every client's Galois keys resolved for every expansion level, before
// any group is enqueued: a failure leaves the caller's stream and `out` untouched, and its message names the client
// by its index in the call.
int32_t check_clients_args(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                           const hecuda_pir_database *const *dbs, int32_t db_count, const int32_t *dims, int32_t dim_count,
                           int32_t chunk_count, const uint64_t *queries, int32_t query_ct_count, int32_t indices_count,
                           const void *out, ResponseShape &shape) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!evks) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (client_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "client_count must be at least 1");
    for (int32_t j = 0; j < client_count; ++j) {
        rc = check_response_args(h, evks[j], dbs, db_count, dims, dim_count, chunk_count, queries, query_ct_count,
                                 indices_count, out, shape);
        if (rc) return fail(rc, "client " + std::to_string(j) + ": " + last_error_cstr());
    }
    const ExpandPlan plan = build_expand_plan(h->ctx->n, query_ct_count, shape.expanded_query_count * indices_count);
    std::vector<LevelKeys> level_keys;
    return resolve_level_keys(evks, client_count, 0, h->ctx->n, plan, level_keys);
}

// PirUtil.computeResponse (PirUtil.swift:490-568) for `clients` (<= HECUDA_MULPIR_CLIENT_GROUP) queries of the same
// shape, client j with keys[j]: d_query = clients x query_ct_count ciphertexts (Coeff), d_out = clients x indices_count x
// chunk_count ciphertexts of 2 x 1 x N (Coeff, one modulus).  Each stage is one pass over all clients; the first
// dimension streams every database once for the whole group.  A group of one keeps the single-client kernels: its
// forward NTT covers only the first-dimension slice of each index, the scan is the single-client scan, and the
// relinearization reads one key instead of a key table.
// first_client: the call-wide index of keys[0] (the keys were resolved by check_clients_args); < 0 for a single-client
// call, whose errors name no client.
int32_t respond_group(const hecuda_context *h, const hecuda_evk *const *keys, int clients, int first_client,
                      const hecuda_pir_database *const *dbs, int32_t db_count, const ResponseShape &shape, const u64 *d_query,
                      int64_t query_ct_count, int64_t indices_count, u64 *d_out, cudaStream_t s) {
    const Context &c = *h->ctx;
    const int L = c.L;
    const int64_t n = c.n;
    const size_t ct_words = (size_t)2 * L * n, reply_words = (size_t)2 * n * shape.chunk_count;
    const int64_t eqc = shape.expanded_query_count, dim0 = shape.dims[0];
    const int64_t rows = shape.chunk_count * shape.columns;  // first-dimension inner products per query
    const int64_t client_cts = eqc * indices_count;            // expanded ciphertexts per client
    // the replies of index qi go straight to `out` unless several clients' replies interleave with other indices'
    const bool direct = clients == 1 || indices_count == 1;
    StreamBuffers tmp(s);
    u64 *expanded = nullptr, *query_eval = nullptr, *results[2] = {nullptr, nullptr}, *lhs = nullptr, *ct3 = nullptr,
        *scratch = nullptr, *replies = nullptr;
    CK(tmp.alloc(&expanded, ct_words * client_cts * clients));
    int32_t rc = expand_device(h, keys, clients, d_query, query_ct_count, client_cts, expanded, s, first_client);
    if (rc) return rc;
    // firstDimensionQueries: convertToEvalFormat (:523-532).  One client transforms only each index's first-dimension
    // slice, into a buffer of dims[0] ciphertexts: captured graphs pin their temporaries, and the slice is 437 of 512
    // ciphertexts at the C4 shape.  A group transforms all its expanded ciphertexts in one launch: the slices of later
    // dimensions (~15 % of this NTT at the C4 shape) are transformed for nothing, which moves fewer bytes than
    // gathering the first-dimension slices into a contiguous buffer would.
    CK(tmp.alloc(&query_eval, clients == 1 ? ct_words * dim0 : ct_words * client_cts * clients));
    CK(tmp.alloc(&results[0], ct_words * rows * clients));
    CK(tmp.alloc(&results[1], ct_words * rows * clients));
    if (!direct) CK(tmp.alloc(&replies, reply_words * clients));
    size_t scratch_words = 0, lhs_words = 0, ct3_words = 0;
    {
        int64_t count = rows;
        for (size_t d = 1; d < shape.dims.size(); ++d) {
            const int64_t size = shape.dims[d], groups = count / size;
            scratch_words = std::max(scratch_words, inner_product_scratch_words(c, size) * (size_t)(groups * clients));
            scratch_words = std::max(scratch_words, relinearize_scratch_words(c, L) * (size_t)(groups * clients));
            lhs_words = std::max(lhs_words, ct_words * (size_t)(size * groups * clients));
            ct3_words = std::max(ct3_words, (size_t)3 * L * n * groups * clients);
            count = groups;
        }
    }
    CK(tmp.alloc(&scratch, scratch_words));
    CK(tmp.alloc(&lhs, lhs_words));
    CK(tmp.alloc(&ct3, ct3_words));
    KsKeyTable relin{};
    for (int j = 0; j < clients; ++j) relin.key[j] = keys[j]->d_relin;
    const NttRowMap map = c.map_q(L);
    cudaError_t e;
    if (clients > 1 && (e = launch_ntt_forward(c, map, expanded, query_eval, client_cts * clients * 2 * L, s)) != cudaSuccess)
        return cuda_fail(e, "ntt");
    const size_t client_pitch = ct_words * client_cts * sizeof(u64);
    for (int64_t qi = 0; qi < indices_count; ++qi) {
        const hecuda_pir_database *db = dbs[db_count == 1 ? 0 : qi];
        const u64 *first_eval = clients == 1 ? query_eval : query_eval + ct_words * eqc * qi;
        if (clients == 1 && (e = launch_ntt_forward(c, map, expanded + ct_words * eqc * qi, query_eval, dim0 * 2 * L, s)) != cudaSuccess)
            return cuda_fail(e, "ntt");
        // every column of every chunk for every client: Scheme.innerProduct(ciphertexts:plaintexts:) then
        // convertToCanonicalFormat (:427-435)
        e = launch_inner_product_plain_clients(c, first_eval, (int64_t)ct_words * client_cts, clients, L, dim0, db->d_plain,
                                               db->d_plain32, db->d_present, results[0], (int64_t)ct_words * rows, rows, s);
        if (e != cudaSuccess) return cuda_fail(e, "innerProduct(ciphertexts:plaintexts:)");
        if ((e = launch_ntt_inverse(c, map, results[0], results[0], rows * clients * 2 * L, kScalePlain, s)) != cudaSuccess)
            return cuda_fail(e, "ntt");
        int64_t count = rows, query_start = dim0;
        int cur = 0;
        for (size_t d = 1; d < shape.dims.size(); ++d) {  // remaining dimensions (:447-480)
            const int64_t size = shape.dims[d], groups = count / size;
            const size_t slice = ct_words * size * sizeof(u64);
            for (int64_t g = 0; g < groups; ++g)  // vector0 = the client's query slice, for each of its groups
                CK(cudaMemcpy2DAsync(lhs + ct_words * size * g, slice * groups, expanded + ct_words * (eqc * qi + query_start),
                                     client_pitch, slice, (size_t)clients, cudaMemcpyDeviceToDevice, s));
            if ((e = inner_product_chunk(c, scratch, lhs, results[cur], size, ct3, groups * clients, s)) != cudaSuccess)
                return cuda_fail(e, "innerProduct");
            relin.items_per_client = groups;
            e = clients == 1 ? relinearize_chunk(c, scratch, keys[0]->d_relin, ct3, L, results[cur ^ 1], groups, s)
                             : relinearize_chunk(c, scratch, nullptr, ct3, L, results[cur ^ 1], groups * clients, s, &relin);
            if (e != cudaSuccess) return cuda_fail(e, "relinearize");
            cur ^= 1;
            count = groups;
            query_start += size;
        }
        if (count != shape.chunk_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "There should be only 1 ciphertext in the final result for each chunk");
        // modSwitchDownToSingle (HeScheme.swift:1481-1485); BFV's canonical format is already Coeff
        u64 *out = d_out + reply_words * qi;
        const u64 *single = results[cur];
        for (int l = L; l > 1; --l) {
            u64 *dst = l > 2 ? results[cur ^ 1] : direct ? out : replies;
            if ((e = launch_mod_switch(c, results[cur], l, dst, count * 2 * clients, s)) != cudaSuccess)
                return cuda_fail(e, "modSwitchDown");
            cur ^= 1;
            single = dst;
        }
        if (single != out)  // one modulus already, or the staged replies of several clients and indices
            CK(cudaMemcpy2DAsync(out, reply_words * indices_count * sizeof(u64), single, reply_words * sizeof(u64),
                                 reply_words * sizeof(u64), (size_t)clients, cudaMemcpyDeviceToDevice, s));
    }
    return HECUDA_OK;
}

// ---------------------------------------------------------------- captured response pipelines
// One query is ~100 small launches (level-by-level expansion, first-dimension scan, ct x ct folding, modulus switches);
// at PIR sizes each kernel runs for a few microseconds, so the call is bound by launch latency.  The host entry point
// therefore captures the pipeline of a (database, evaluation key, shape) triple into a CUDA graph the first time it
// sees it and replays it afterwards: one graph launch per query.  An instance owns its query / reply buffers (the
// addresses are baked into the graph) and serves one query at a time; concurrent callers get instances of their own.
}  // namespace
namespace hecuda {
namespace api {
struct PirGraph {
    const hecuda_evk *evk = nullptr;
    unsigned long long evk_version = 0;
    const hecuda_pir_database *db = nullptr;
    std::vector<int64_t> dims;
    int64_t chunk_count = 0, query_ct_count = 0;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    u64 *d_query = nullptr, *d_out = nullptr;
    unsigned long long launches = 0;  // kernels inside the graph (for hecuda_kernel_launch_count)
    bool busy = false;
    void release() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        if (d_query) cudaFree(d_query);
        if (d_out) cudaFree(d_out);
    }
};
// Handles may outlive their context (a garbage-collected host destroys them in any order): only touch a live context.
static std::mutex g_live_mu;
static std::set<const hecuda_context *> g_live;
void context_registered(const hecuda_context *h, bool alive) {
    std::lock_guard<std::mutex> lock(g_live_mu);
    if (alive) g_live.insert(h);
    else g_live.erase(h);
}
void pir_graphs_purge(hecuda_context *h, const void *handle) {
    if (!h) return;
    std::vector<PirGraph *> dead;
    {
        std::lock_guard<std::mutex> live(g_live_mu);
        if (!g_live.count(h)) return;
        std::lock_guard<std::mutex> lock(h->mu);
        auto &v = h->pir_graphs;
        for (size_t i = 0; i < v.size();) {
            if (!handle || v[i]->evk == handle || v[i]->db == handle) {
                dead.push_back(v[i]);
                v.erase(v.begin() + (long)i);
            } else {
                ++i;
            }
        }
    }
    if (!dead.empty()) cudaDeviceSynchronize();  // a purged instance may still be replaying on another thread's stream
    for (PirGraph *g : dead) {
        g->release();
        delete g;
    }
}
}  // namespace api
}  // namespace hecuda
namespace {

// Finds an idle instance for this call or builds one; nullptr (with *rc == OK) when capture is not possible.
PirGraph *acquire_graph(const hecuda_context *hc, const hecuda_evk *k, const hecuda_pir_database *db, const ResponseShape &shape,
                        int64_t query_ct_count, cudaStream_t s, int32_t *rc) {
    hecuda_context *h = const_cast<hecuda_context *>(hc);
    *rc = HECUDA_OK;
    {
        std::lock_guard<std::mutex> lock(h->mu);
        for (PirGraph *g : h->pir_graphs)
            if (!g->busy && g->evk == k && g->evk_version == k->version && g->db == db && g->dims == shape.dims &&
                g->chunk_count == shape.chunk_count && g->query_ct_count == query_ct_count) {
                g->busy = true;
                return g;
            }
    }
    const Context &c = *h->ctx;
    // the shape's expansion plan goes to the context's cache before the capture: a miss inside it would allocate and
    // copy synchronously, which invalidates the capture
    const ExpandStep *d_steps = nullptr;
    if ((*rc = expand_steps_on_device(hc, c.n, query_ct_count, shape.expanded_query_count, &d_steps))) return nullptr;
    const size_t ct_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * c.n * shape.chunk_count;
    PirGraph *g = new (std::nothrow) PirGraph();
    if (!g) return nullptr;
    g->evk = k;
    g->evk_version = k->version;
    g->db = db;
    g->dims = shape.dims;
    g->chunk_count = shape.chunk_count;
    g->query_ct_count = query_ct_count;
    cudaError_t e = cudaMalloc(&g->d_query, ct_words * query_ct_count * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&g->d_out, out_words * sizeof(u64));
    if (e != cudaSuccess) {
        g->release();
        delete g;
        *rc = cuda_fail(e, "response graph buffers");
        return nullptr;
    }
    e = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
    int32_t body = HECUDA_OK;
    if (e == cudaSuccess) {
        body = respond_group(hc, &k, 1, -1, &db, 1, shape, g->d_query, query_ct_count, 1, g->d_out, s);
        e = cudaStreamEndCapture(s, &g->graph);
    }
    if (e == cudaSuccess && body == HECUDA_OK) e = cudaGraphInstantiate(&g->exec, g->graph, 0);
    if (e == cudaSuccess && body == HECUDA_OK) {  // kernels per replay, for hecuda_kernel_launch_count
        size_t count = 0;
        if (cudaGraphGetNodes(g->graph, nullptr, &count) == cudaSuccess && count) {
            std::vector<cudaGraphNode_t> nodes(count);
            cudaGraphGetNodes(g->graph, nodes.data(), &count);
            for (size_t i = 0; i < count; ++i) {
                cudaGraphNodeType type;
                if (cudaGraphNodeGetType(nodes[i], &type) == cudaSuccess && type == cudaGraphNodeTypeKernel) ++g->launches;
            }
        }
    }
    if (e != cudaSuccess || body != HECUDA_OK) {  // not capturable on this setup: the caller takes the direct path
        cudaGetLastError();
        g->release();
        delete g;
        if (body != HECUDA_OK) *rc = body;
        return nullptr;
    }
    g->busy = true;
    // bounded cache: every instance pins its scratch (tens of MB); beyond the cap the oldest idle one makes room
    const char *cap_env = std::getenv("HECUDA_PIR_GRAPH_CACHE");  // (read per build: building a graph is the slow path)
    const long cap_v = cap_env ? std::atol(cap_env) : 32;
    const size_t cap = (size_t)(cap_v < 1 ? 1 : cap_v);
    PirGraph *evicted = nullptr;
    {
        std::lock_guard<std::mutex> lock(h->mu);
        if (h->pir_graphs.size() >= cap)
            for (size_t i = 0; i < h->pir_graphs.size(); ++i)
                if (!h->pir_graphs[i]->busy) {
                    evicted = h->pir_graphs[i];
                    h->pir_graphs.erase(h->pir_graphs.begin() + (long)i);
                    break;
                }
        h->pir_graphs.push_back(g);
    }
    if (evicted) {  // idle: its last replay was waited for by its caller
        evicted->release();
        delete evicted;
    }
    return g;
}
void release_graph(const hecuda_context *hc, PirGraph *g) {
    hecuda_context *h = const_cast<hecuda_context *>(hc);
    std::lock_guard<std::mutex> lock(h->mu);
    g->busy = false;
}

// ---------------------------------------------------------------- host bodies
// The host calls run client_count clients' queries through one workspace stream, group by group: stage a group's
// queries, answer the group, copy its replies back.  Temporaries are sized for one group.  single: a single-client
// call, whose errors name no client.
int32_t respond_words(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count, bool single,
                      const hecuda_pir_database *const *dbs, int32_t db_count, const ResponseShape &shape,
                      const uint64_t *queries, int32_t query_ct_count, int32_t indices_count, uint64_t *out) {
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    const size_t query_words = (size_t)2 * h->ctx->L * h->ctx->n * query_ct_count;
    const size_t out_words = (size_t)2 * h->ctx->n * shape.chunk_count * indices_count;
    const int group = std::min<int32_t>(HECUDA_MULPIR_CLIENT_GROUP, client_count);
    StreamBuffers tmp(s);
    u64 *d_query = nullptr, *d_out = nullptr;
    CK(tmp.alloc(&d_query, query_words * group));
    CK(tmp.alloc(&d_out, out_words * group));
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    for (int32_t first = 0; first < client_count; first += group) {
        const int clients = std::min<int32_t>(group, client_count - first);
        CK(cudaMemcpyAsync(d_query, queries + query_words * first, query_words * clients * sizeof(u64), cudaMemcpyHostToDevice, s));
        const int32_t rc = respond_group(h, evks + first, clients, single ? -1 : first, dbs, db_count, shape, d_query,
                                         query_ct_count, indices_count, d_out, s);
        if (rc) return rc;
        CK(cudaMemcpyAsync(out + out_words * first, d_out, out_words * clients * sizeof(u64), cudaMemcpyDeviceToHost, s));
    }
    CK(wait_stream(s));
    return HECUDA_OK;
}

// The same with seeded queries in and packed replies out: per group, one seeded expansion of all the group's query
// ciphertexts, the group's responses, and one packing pass per reply poly over the group's replies.
int32_t respond_wire(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count, bool single,
                     const hecuda_pir_database *const *dbs, int32_t db_count, const ResponseShape &shape,
                     const uint8_t *query_poly0, const uint8_t *query_seeds, int32_t query_ct_count, int32_t indices_count,
                     int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint8_t *out) {
    if (!query_seeds) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    WireCodec wc;
    int32_t rc = wc.setup(*h->ctx, skip_lsbs_poly0, skip_lsbs_poly1);
    if (rc) return rc;
    const Context &c = *h->ctx;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    const int group = std::min<int32_t>(HECUDA_MULPIR_CLIENT_GROUP, client_count);
    const size_t ct_words = (size_t)2 * c.L * c.n, poly0_bytes = wc.query_bytes * query_ct_count, seed_bytes = (size_t)32 * query_ct_count;
    const int64_t replies = (int64_t)indices_count * shape.chunk_count;  // per client
    const size_t out_bytes = wc.reply_bytes() * replies;
    unsigned char *d_poly0 = nullptr, *d_seeds = nullptr;
    u64 *d_query = nullptr, *d_resp = nullptr;
    CK(tmp.alloc_bytes((void **)&d_poly0, poly0_bytes * group));
    CK(tmp.alloc_bytes((void **)&d_seeds, seed_bytes * group));
    CK(tmp.alloc(&d_query, ct_words * query_ct_count * group));
    CK(tmp.alloc(&d_resp, (size_t)2 * c.n * replies * group));
    CK(wc.alloc(tmp, c, replies * group));
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    for (int32_t first = 0; first < client_count; first += group) {
        const int clients = std::min<int32_t>(group, client_count - first);
        CK(cudaMemcpyAsync(d_poly0, query_poly0 + poly0_bytes * first, poly0_bytes * clients, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_seeds, query_seeds + seed_bytes * first, seed_bytes * clients, cudaMemcpyHostToDevice, s));
        // Query.ciphertexts arrive as SerializedCiphertext.seeded (SerializedCiphertext.swift:41-49)
        cudaError_t e = expand_seeded_device(c, c.L, d_poly0, d_seeds, d_query, (int64_t)query_ct_count * clients, s);
        if (e != cudaSuccess) return cuda_fail(e, "expand seeded query");
        rc = respond_group(h, evks + first, clients, single ? -1 : first, dbs, db_count, shape, d_query, query_ct_count,
                           indices_count, d_resp, s);
        if (rc) return rc;
        // the group's replies are client-major, like `out`
        if ((rc = wc.pack(c, d_resp, replies * clients, s))) return rc;
        CK(cudaMemcpyAsync(out + out_bytes * first, wc.reply, out_bytes * clients, cudaMemcpyDeviceToHost, s));
    }
    CK(wait_stream(s));
    return HECUDA_OK;
}

// ---------------------------------------------------------------- protobuf messages in and out
// respond_wire with EncryptedIndices messages in and PIRResponse messages out.  Per group: the group's messages
// uploaded back to back, the seeded expansion reading poly0 and the seeds in place (and the .full query ciphertexts
// loaded over theirs), the group's responses, then each reply ciphertext packed straight into its slot of its client's
// PIRResponse with one framing launch and one packing launch per reply poly.
int32_t respond_proto(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                      const hecuda_pir_database *const *dbs, int32_t db_count, const ResponseShape &shape,
                      const uint8_t *const *messages, const uint64_t *message_byte_counts,
                      const std::vector<pirproto::Query> &queries, int32_t query_ct_count, int32_t indices_count,
                      int32_t skip0, int32_t skip1, const pirproto::ResponseLayout &rl, uint8_t *out) {
    WireCodec wc;
    int32_t rc = wc.setup(*h->ctx, skip0, skip1);
    if (rc) return rc;
    const Context &c = *h->ctx;
    FrameRuns frame;  // every reply ciphertext's framing (and its reply's opening before its first one)
    frame.size = rl.size;
    for (long long r = 0; r < rl.indices * rl.chunks; ++r)
        rl.frame(r, [&](long long at, const pirproto::Bytes &b) { frame.put(at, b); });
    const int group = std::min<int32_t>(HECUDA_MULPIR_CLIENT_GROUP, client_count);
    const int64_t replies = (int64_t)indices_count * shape.chunk_count;  // per client
    const size_t ct_words = (size_t)2 * c.L * c.n;
    size_t msg_bytes = 0;
    for (int32_t first = 0; first < client_count; first += group) {
        size_t bytes = 0;
        for (int32_t j = first; j < std::min<int32_t>(first + group, client_count); ++j) bytes += message_byte_counts[j];
        msg_bytes = std::max(msg_bytes, bytes);
    }
    // reply ciphertext k of a group (client-major) is polys 2k, 2k + 1 of the group's responses; its poly p goes to
    // byte tag[p][k] of the group's PIRResponses
    std::vector<long long> pack((size_t)4 * (group * replies + 1));
    for (int p = 0; p < 2; ++p) {
        long long *tag = pack.data() + (size_t)2 * p * (group * replies + 1), *slot = tag + group * replies + 1;
        for (int64_t k = 0; k < group * replies; ++k) {
            tag[k] = (k / replies) * rl.size + rl.poly_at(k % replies, p);
            slot[k] = 2 * k + p;
        }
        tag[group * replies] = group * rl.size;
    }
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    unsigned char *d_msg = nullptr, *d_out = nullptr;
    u64 *d_query = nullptr, *d_resp = nullptr;
    long long *d_pack = nullptr, *d_tables = nullptr, *d_runs = nullptr;
    unsigned char *d_frame = nullptr;
    const size_t table_words = (size_t)2 * query_ct_count * group + 1 + (size_t)6 * query_ct_count * group;
    CK(tmp.alloc_bytes((void **)&d_msg, msg_bytes + 32));  // + 32 zero bytes: the seed a .full ciphertext expands
    CK(tmp.alloc(&d_query, ct_words * query_ct_count * group));
    CK(tmp.alloc(&d_resp, (size_t)2 * c.n * replies * group));
    CK(tmp.alloc_bytes((void **)&d_out, (size_t)rl.size * group));
    CK(tmp.alloc_bytes((void **)&d_pack, pack.size() * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_tables, table_words * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_runs, frame.table.size() * sizeof(long long)));
    CK(tmp.alloc_bytes((void **)&d_frame, frame.bytes.size()));
    CodecConsts full_cc;
    std::string err;
    std::vector<std::vector<long long>> staged;  // host tables stay alive until the stream is drained
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    CK(cudaMemcpyAsync(d_pack, pack.data(), pack.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_runs, frame.table.data(), frame.table.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_frame, frame.bytes.data(), frame.bytes.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(d_msg + msg_bytes, 0, 32, s));
    for (int32_t first = 0; first < client_count; first += group) {
        const int clients = std::min<int32_t>(group, client_count - first);
        std::vector<long long> msg_at((size_t)clients);
        long long at = 0;
        for (int j = 0; j < clients; ++j) {
            msg_at[(size_t)j] = at;
            CK(cudaMemcpyAsync(d_msg + at, messages[first + j], message_byte_counts[first + j], cudaMemcpyHostToDevice, s));
            at += (long long)message_byte_counts[first + j];
        }
        std::vector<const std::vector<pirproto::Ciphertext> *> cts_of((size_t)clients);
        for (int j = 0; j < clients; ++j) cts_of[(size_t)j] = &queries[(size_t)(first + j)].cts;
        const GroupTables t = group_tables(cts_of, msg_at, (long long)msg_bytes);
        staged.emplace_back(t.tag);
        std::vector<long long> &flat = staged.back();
        flat.insert(flat.end(), t.seed.begin(), t.seed.end());
        for (const auto &f : t.full) flat.insert(flat.end(), f.second.begin(), f.second.end());
        CK(cudaMemcpyAsync(d_tables, flat.data(), flat.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
        PolyLayout seeded;
        seeded.tag = d_tables, seeded.seed = d_tables + t.tag.size(), seeded.frame = 0;
        const int64_t batch = (int64_t)query_ct_count * clients;
        cudaError_t e = expand_seeded_device(c, c.L, d_msg, nullptr, d_query, batch, s, seeded);
        if (e != cudaSuccess) return cuda_fail(e, "expand seeded query");
        // .full query ciphertexts (Ciphertext(deserialize:) of .full): both polys over the zero rows expanded above
        const long long *table = seeded.seed + t.seed.size();
        for (const auto &f : t.full) {
            const int64_t count = (int64_t)(f.second.size() - 1) / 2;
            if (!codec_consts(c, c.map_q(c.L), f.first, full_cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
            PolyLayout full;
            full.tag = table, full.slot = table + count + 1, full.frame = 0;
            if ((e = launch_poly_load(c, full_cc, f.first, d_msg, d_query, count, s, full)) != cudaSuccess)
                return cuda_fail(e, "load full query ciphertexts");
            table += f.second.size();
        }
        rc = respond_group(h, evks + first, clients, first, dbs, db_count, shape, d_query, query_ct_count, indices_count,
                           d_resp, s);
        if (rc) return rc;
        const int64_t cts = replies * clients;
        if ((e = launch_frame_runs(d_out, clients, rl.size, d_runs, frame.runs(), d_frame, s)) != cudaSuccess)
            return cuda_fail(e, "frame response");
        for (int p = 0; p < 2; ++p) {
            PolyLayout at;
            at.tag = d_pack + (size_t)2 * p * (group * replies + 1), at.slot = at.tag + group * replies + 1, at.frame = 0;
            if ((e = launch_poly_serialize(c, wc.out[p], wc.skip[p], d_resp, d_out, cts, s, at)) != cudaSuccess)
                return cuda_fail(e, "serialize response");
        }
        CK(cudaMemcpyAsync(out + (size_t)rl.size * first, d_out, (size_t)rl.size * clients, cudaMemcpyDeviceToHost, s));
    }
    CK(wait_stream(s));
    return HECUDA_OK;
}

// Small moduli (the default PIR parameters): keep the rows as uint32 -- half the bytes per scan, half the HBM
cudaError_t narrow_database(const Context &c, hecuda_pir_database *db) {
    if (!inner_product_plain_small_supported(c, c.L)) return cudaSuccess;
    const size_t words = (size_t)c.L * c.n * db->count;
    cudaError_t e = cudaMalloc(&db->d_plain32, words * sizeof(u32));
    if (e == cudaSuccess) e = launch_narrow(db->d_plain, db->d_plain32, (int64_t)words, nullptr);
    if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
    if (e == cudaSuccess) {
        cudaFree(db->d_plain);
        db->d_plain = nullptr;
    }
    return e;
}

std::string describe(const char *fmt, long long a, long long b) {
    char buf[160];
    snprintf(buf, sizeof buf, fmt, a, b);
    return buf;
}

// MulPirServer.process's arguments (MulPir.swift:433-556; the checks of hecuda/pir.py plaintextRows), all on the
// host: on success `s` describes the database except for its device pointers, `bytes` is how many entry bytes to
// upload and `count` = chunkCount * prod(dimensions).
int32_t pir_process_shape(const hecuda_context *h, const uint8_t *entries, const uint64_t *offsets, int64_t entry_count,
                          int64_t entry_size, int32_t encode_entry_size, const int32_t *dims, int32_t dim_count,
                          procdb::PirShape &s, size_t &bytes, int64_t &count) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!entries || !dims) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (dim_count != 1 && dim_count != 2)
        return fail(HECUDA_ERR_INVALID_ARGUMENT,
                    "invalidDimensionCount(dimensionCount: " + std::to_string(dim_count) + ", expected: [1, 2])");
    if (entry_count < 0 || entry_size < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "negative entry count / empty entry size");
    int64_t per_chunk = 1;
    for (int i = 0; i < dim_count; ++i) {
        if (dims[i] < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "dimensions must be positive");
        per_chunk *= dims[i];
    }
    const Context &c = *h->ctx;
    s = procdb::pir_shape(c.n, c.t, entry_count, entry_size, encode_entry_size != 0, per_chunk, dims[0]);
    if (s.bits < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "plaintext modulus below 2");
    int64_t longest = entry_count ? entry_size : 0;
    if (offsets) {
        longest = 0;
        for (int64_t i = 0; i < entry_count; ++i) {
            if (offsets[i + 1] < offsets[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "offsets must not decrease");
            longest = std::max<int64_t>(longest, (int64_t)(offsets[i + 1] - offsets[i]));
        }
        bytes = (size_t)offsets[entry_count];
    } else {
        bytes = (size_t)(entry_count * entry_size);
    }
    if (longest > entry_size)
        return fail(HECUDA_ERR_INVALID_ARGUMENT,
                    describe("invalidDatabaseEntrySize(maximumEntrySize: %lld, expected: %lld)", longest, entry_size));
    const int64_t chunks = procdb::pir_chunk_count(s);
    if (chunks > 1) {  // processSplitLargeEntries: one entry per plaintext and chunk
        if (entry_count > per_chunk)
            return fail(HECUDA_ERR_INVALID_ARGUMENT,
                        describe("invalidDatabaseEntryCount(entryCount: %lld, expected: at most %lld)", entry_count, per_chunk));
    } else {  // processPackEntries
        const int64_t pieces = (entry_count * s.encoded + s.stride - 1) / s.stride;
        if (pieces > per_chunk)
            return fail(HECUDA_ERR_INVALID_ARGUMENT,
                        describe("invalidDatabaseEntryCount(entryCount: %lld, expected: at most %lld)", entry_count,
                               per_chunk * (s.stride / s.encoded)));
    }
    count = chunks * per_chunk;
    return HECUDA_OK;
}

// Packs the `count` plaintexts of a database whose entry bytes (and offsets) are already on the device (`s` holds the
// device pointers) slab by slab on the default stream: present flags into d_present[count], each slab's coefficients
// handed to sink(first, items, d_coeff).
template <class Sink>
cudaError_t pir_pack_device_slabs(const Context &c, const procdb::PirShape &s, int64_t count, unsigned char *d_present,
                                  Sink sink) {
    u64 *d_coeff = nullptr;
    const int64_t slab = coefficient_slab(c);
    cudaError_t e = cudaMalloc(&d_coeff, (size_t)std::max<int64_t>(1, std::min(slab, count)) * c.n * sizeof(u64));
    for (int64_t done = 0; e == cudaSuccess && done < count; done += slab) {
        const int64_t items = std::min(slab, count - done);
        e = launch_pir_pack(s, (int)c.n, done, items, d_coeff, d_present + done, nullptr);
        if (e == cudaSuccess) e = sink(done, items, d_coeff);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
    cudaFree(d_coeff);
    return e;
}

// Uploads the entry bytes (and offsets) once, then packs them with pir_pack_device_slabs.  Frees its buffers before it
// returns.
template <class Sink>
cudaError_t pir_pack_slabs(const Context &c, procdb::PirShape s, const uint8_t *entries, const uint64_t *offsets,
                           size_t bytes, int64_t count, unsigned char *d_present, Sink sink) {
    unsigned char *d_entries = nullptr;
    uint64_t *d_offsets = nullptr;
    cudaError_t e = cudaMalloc(&d_entries, std::max<size_t>(bytes, 1));
    if (e == cudaSuccess && bytes) e = upload(d_entries, entries, bytes);
    if (e == cudaSuccess && offsets) {
        const size_t offset_bytes = (size_t)(s.entry_count + 1) * sizeof(uint64_t);
        e = cudaMalloc(&d_offsets, offset_bytes);
        if (e == cudaSuccess) e = upload(d_offsets, offsets, offset_bytes);
    }
    s.entries = d_entries;
    s.offsets = d_offsets;
    if (e == cudaSuccess) e = pir_pack_device_slabs(c, s, count, d_present, sink);
    cudaFree(d_offsets);
    cudaFree(d_entries);
    return e;
}

// Plaintext.convertToEvalFormat (Plaintext.swift:149-171) of every packed slab, straight into the database's rows
cudaError_t pir_fill_database(const Context &c, const procdb::PirShape &device_shape, hecuda_pir_database *db) {
    const size_t row_words = (size_t)c.L * c.n;
    cudaError_t e = cudaMalloc(&db->d_plain, row_words * db->count * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&db->d_present, (size_t)db->count);
    if (e == cudaSuccess)
        e = pir_pack_device_slabs(c, device_shape, db->count, db->d_present, [&](int64_t first, int64_t items, const u64 *d) {
            return launch_plaintext_to_eval(c, d, c.L, db->d_plain + row_words * first, items, nullptr);
        });
    return e;
}

}  // namespace

namespace hecuda {
namespace api {

// hecuda_keyword_pir_databases_create's databases (keyword_pir.cu): `tables` MulPir databases, table t made of entries
// [t * per_table, (t + 1) * per_table) of device bytes d_entries with global offsets (h_offsets on the host, d_offsets
// on the device).  Each database is word for word what hecuda_pir_database_create_from_entries builds from the same
// entries with encode_entry_size = 0.  On error every out[t] is NULL and nothing stays allocated.
int32_t pir_databases_from_device_entries(const hecuda_context *h, const unsigned char *d_entries, const uint64_t *h_offsets,
                                          const uint64_t *d_offsets, int64_t per_table, int tables, int64_t entry_size,
                                          const int32_t *dims, int32_t dim_count, hecuda_pir_database **out) {
    for (int t = 0; t < tables; ++t) out[t] = nullptr;
    std::vector<procdb::PirShape> shapes((size_t)tables);
    int64_t count = 0;
    for (int t = 0; t < tables; ++t) {
        size_t bytes = 0;
        int32_t rc = pir_process_shape(h, d_entries, h_offsets + (size_t)t * per_table, per_table, entry_size, 0, dims,
                                       dim_count, shapes[t], bytes, count);
        if (rc) return rc;
        shapes[t].entries = d_entries;
        shapes[t].offsets = d_offsets + (size_t)t * per_table;
    }
    const Context &c = *h->ctx;
    cudaError_t e = cudaSuccess;
    for (int t = 0; t < tables && e == cudaSuccess; ++t) {
        hecuda_pir_database *db = new (std::nothrow) hecuda_pir_database();
        if (!db) {
            e = cudaErrorMemoryAllocation;
            break;
        }
        db->owner = h;
        db->count = count;
        out[t] = db;
        e = pir_fill_database(c, shapes[t], db);
        if (e == cudaSuccess) e = narrow_database(c, db);
    }
    if (e != cudaSuccess) {
        for (int t = 0; t < tables; ++t) {
            if (out[t]) hecuda_pir_database_destroy(out[t]);
            out[t] = nullptr;
        }
        return cuda_fail(e, "keyword pir databases");
    }
    return HECUDA_OK;
}

}  // namespace api
}  // namespace hecuda

// ---------------------------------------------------------------- saving and loading processed databases
// ProcessedDatabase.serialize / init(from:context:) (IndexPirProtocol.swift:286-378).  The host walks the tags
// (database_io.hpp); whole plaintexts then cross PCIe in chunks of at most one 64 MB slab through two device staging
// buffers, one stream each, so that chunk k + 1's copy runs under chunk k's kernel.  The kernels (codec.cu) unpack
// straight into the resident rows, or pack straight from them.
namespace {

// one chunk of the pipeline: plaintexts of the stream, the first of which is plaintext `local` of database `db`
struct DbChunk {
    int db;
    int64_t local;
    dbio::Chunk chunk;
};

// the chunks of databases of counts[t] plaintexts each, concatenated in the stream, and the largest chunk's bytes
std::vector<DbChunk> plan_db_chunks(const std::vector<long long> &tag, const std::vector<int64_t> &counts, long long &widest) {
    std::vector<DbChunk> plan;
    widest = 1;
    int64_t first = 0;
    for (size_t t = 0; t < counts.size(); first += counts[t++])
        for (const dbio::Chunk &ch : dbio::plan_chunks(tag, first, first + counts[t], kSlabBytes)) {
            plan.push_back({(int)t, ch.first - first, ch});
            widest = std::max(widest, tag[(size_t)(ch.first + ch.count)] - tag[(size_t)ch.first]);
        }
    return plan;
}

// resident rows of a database, whichever word type it keeps
struct ResidentRows {
    u64 *p64;
    u32 *p32;
    size_t row_words;
    template <class F>
    cudaError_t with(int64_t first, F f) const {
        return p32 ? f(p32 + row_words * first) : f(p64 + row_words * first);
    }
};
ResidentRows resident_rows(const Context &c, const hecuda_pir_database *db) {
    return {db->d_plain, db->d_plain32, (size_t)c.L * c.n};
}

std::string corrupted(const std::string &what) { return "corruptedData(" + what + ")"; }

int32_t load_refusal(const dbio::TagWalk &w, uint64_t byte_count, long long plaintext_bytes) {
    const std::string size = std::to_string(byte_count) + "-byte buffer";
    switch (w.error) {
    case dbio::TagWalk::kVersion:
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidDatabaseSerializationVersion(serializationVersion: " +
                                                     std::to_string(w.value) + ", expected: " + std::to_string(dbio::kVersion) + ")");
    case dbio::TagWalk::kTag:
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidDatabaseSerializationPlaintextTag(tag: " + std::to_string(w.value) +
                                                     ") of plaintext " + std::to_string(w.at));
    default:
        if (w.at < 0 && w.count == 0)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, corrupted("the header runs past the end of the " + size));
        if (w.at < 0)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, corrupted("plaintextCount " + std::to_string(w.count) + " cannot fit the " + size));
        return fail(HECUDA_ERR_INVALID_ARGUMENT, corrupted("plaintext " + std::to_string(w.at) + " (" +
                                                           std::to_string(plaintext_bytes) + " bytes after its tag) runs past the end of the " + size));
    }
}

// The checks shared by the byte count and the serialization, and the tag offset of every plaintext of the
// concatenated databases.  Copies the presence flags to the host; launches nothing.
int32_t serialization_plan(const hecuda_pir_database *const *dbs, int32_t database_count, CodecConsts &cc,
                           std::vector<long long> &tag) {
    if (!dbs || database_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / no databases");
    long long total = 0;
    for (int32_t i = 0; i < database_count; ++i) {
        if (!dbs[i]) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null database");
        if (dbs[i]->owner != dbs[0]->owner)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidContext: the databases belong to different contexts");
        total += dbs[i]->count;
    }
    int32_t rc = check_ctx(dbs[0]->owner);
    if (rc) return rc;
    if (total > dbio::kMaxCount)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "a serialized database holds at most 2^32 - 1 plaintexts (UInt32 plaintextCount), not " +
                                                     std::to_string(total));
    const Context &c = *dbs[0]->owner->ctx;
    std::string err;
    if (!codec_consts(c, c.map_q(c.L), 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    std::vector<unsigned char> present((size_t)total);
    long long at = 0;
    for (int32_t i = 0; i < database_count; ++i) {
        if (dbs[i]->d_present)
            CK(cudaMemcpy(present.data() + at, dbs[i]->d_present, (size_t)dbs[i]->count, cudaMemcpyDeviceToHost));
        else
            memset(present.data() + at, 1, (size_t)dbs[i]->count);
        at += dbs[i]->count;
    }
    if (std::find(present.begin(), present.end(), 1) == present.end()) return fail(HECUDA_ERR_INVALID_ARGUMENT, "emptyDatabase");
    dbio::tag_offsets(present.data(), total, serialized_poly_bytes(cc), tag);
    return HECUDA_OK;
}

}  // namespace

extern "C" {

int32_t hecuda_pir_process_entries(const hecuda_context *h, const uint8_t *entries, const uint64_t *offsets,
                                   int64_t entry_count, int64_t entry_size, int32_t encode_entry_size, const int32_t *dims,
                                   int32_t dim_count, uint64_t *plaintexts, uint8_t *present, int64_t count) {
    procdb::PirShape s;
    size_t bytes = 0;
    int64_t expected = 0;
    int32_t rc = pir_process_shape(h, entries, offsets, entry_count, entry_size, encode_entry_size, dims, dim_count, s,
                                   bytes, expected);
    if (rc) return rc;
    if (!plaintexts || !present) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (count != expected)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, describe("count %lld != chunkCount * prod(dimensions) = %lld", count, expected));
    const Context &c = *h->ctx;
    unsigned char *d_present = nullptr;
    cudaError_t e = cudaMalloc(&d_present, (size_t)count);
    if (e == cudaSuccess)
        e = pir_pack_slabs(c, s, entries, offsets, bytes, count, d_present, [&](int64_t first, int64_t items, const u64 *d) {
            return cudaMemcpy(plaintexts + (size_t)first * c.n, d, (size_t)items * c.n * sizeof(u64), cudaMemcpyDeviceToHost);
        });
    if (e == cudaSuccess) e = cudaMemcpy(present, d_present, (size_t)count, cudaMemcpyDeviceToHost);
    cudaFree(d_present);
    return e == cudaSuccess ? HECUDA_OK : cuda_fail(e, "pir process entries");
}

int32_t hecuda_pir_database_create_from_entries(const hecuda_context *h, const uint8_t *entries, const uint64_t *offsets,
                                                int64_t entry_count, int64_t entry_size, int32_t encode_entry_size,
                                                const int32_t *dims, int32_t dim_count, hecuda_pir_database **out) {
    if (!out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    procdb::PirShape s;
    size_t bytes = 0;
    int64_t count = 0;
    int32_t rc = pir_process_shape(h, entries, offsets, entry_count, entry_size, encode_entry_size, dims, dim_count, s,
                                   bytes, count);
    if (rc) return rc;
    const Context &c = *h->ctx;
    hecuda_pir_database *db = new (std::nothrow) hecuda_pir_database();
    if (!db) return fail(HECUDA_ERR_CUDA, "out of host memory");
    db->owner = h;
    db->count = count;
    unsigned char *d_entries = nullptr;
    uint64_t *d_offsets = nullptr;
    cudaError_t e = cudaMalloc(&d_entries, std::max<size_t>(bytes, 1));
    if (e == cudaSuccess && bytes) e = upload(d_entries, entries, bytes);
    if (e == cudaSuccess && offsets) {
        const size_t offset_bytes = (size_t)(entry_count + 1) * sizeof(uint64_t);
        e = cudaMalloc(&d_offsets, offset_bytes);
        if (e == cudaSuccess) e = upload(d_offsets, offsets, offset_bytes);
    }
    s.entries = d_entries;
    s.offsets = d_offsets;
    if (e == cudaSuccess) e = pir_fill_database(c, s, db);  // one slab at a time
    cudaFree(d_offsets);
    cudaFree(d_entries);
    if (e == cudaSuccess) e = narrow_database(c, db);
    if (e != cudaSuccess) {
        hecuda_pir_database_destroy(db);
        return cuda_fail(e, "pir database from entries");
    }
    *out = db;
    return HECUDA_OK;
}

int32_t hecuda_pir_database_create(const hecuda_context *h, const uint64_t *plaintexts, int32_t eval_format,
                                   const uint8_t *present, int64_t count, hecuda_pir_database **out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!out || !plaintexts || count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / empty database");
    *out = nullptr;
    const Context &c = *h->ctx;
    const size_t row_words = (size_t)c.L * c.n;
    hecuda_pir_database *db = new (std::nothrow) hecuda_pir_database();
    if (!db) return fail(HECUDA_ERR_CUDA, "out of host memory");
    db->owner = h;
    db->count = count;
    cudaError_t e = cudaMalloc(&db->d_plain, row_words * count * sizeof(u64));
    if (e == cudaSuccess && present) {  // no flags at all = every plaintext present: the scan then runs without the test
        e = cudaMalloc(&db->d_present, (size_t)count);
        if (e == cudaSuccess) e = upload(db->d_present, present, (size_t)count);
    }
    if (e == cudaSuccess) {
        if (eval_format) {
            e = upload(db->d_plain, plaintexts, row_words * count * sizeof(u64));
        } else {  // Plaintext.convertToEvalFormat (Plaintext.swift:149-171) in slabs of <= 64 MB of coefficients
            const int64_t slab = coefficient_slab(c);
            u64 *d_coeff = nullptr;
            e = cudaMalloc(&d_coeff, (size_t)std::min(slab, count) * c.n * sizeof(u64));
            for (int64_t done = 0; e == cudaSuccess && done < count; done += slab) {
                const int64_t items = std::min(slab, count - done);
                e = upload(d_coeff, plaintexts + (size_t)done * c.n, (size_t)items * c.n * sizeof(u64));
                if (e == cudaSuccess) e = launch_plaintext_to_eval(c, d_coeff, c.L, db->d_plain + row_words * done, items, nullptr);
                if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
            }
            cudaFree(d_coeff);
        }
    }
    if (e == cudaSuccess) e = narrow_database(c, db);
    if (e != cudaSuccess) {
        hecuda_pir_database_destroy(db);
        return cuda_fail(e, "pir database upload");
    }
    *out = db;
    return HECUDA_OK;
}

int32_t hecuda_pir_database_destroy(hecuda_pir_database *db) {
    if (!db) return HECUDA_OK;
    if (db->owner) pir_graphs_purge(const_cast<hecuda_context *>(db->owner), db);
    if (db->d_plain) cudaFree(db->d_plain);
    if (db->d_plain32) cudaFree(db->d_plain32);
    if (db->d_present) cudaFree(db->d_present);
    delete db;
    return HECUDA_OK;
}

int32_t hecuda_pir_database_device_buffer(hecuda_pir_database *db, void **device_ptr, uint64_t *bytes) {
    if (!db || !device_ptr || !bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    // (uint32 rows when every ciphertext modulus is below 2^31: the bytes say which)
    *device_ptr = db->d_plain32 ? (void *)db->d_plain32 : (void *)db->d_plain;
    *bytes = (uint64_t)db->count * db->owner->ctx->L * db->owner->ctx->n * (db->d_plain32 ? sizeof(u32) : sizeof(u64));
    return HECUDA_OK;
}

int32_t hecuda_pir_database_present(const hecuda_pir_database *db, uint8_t *out, int64_t capacity) {
    if (!db || !out) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    if (capacity < db->count) return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity below the plaintext count");
    if (!db->d_present) {
        memset(out, 1, (size_t)db->count);
        return HECUDA_OK;
    }
    CK(cudaMemcpy(out, db->d_present, (size_t)db->count, cudaMemcpyDeviceToHost));
    return HECUDA_OK;
}

int32_t hecuda_pir_databases_create_serialized(const hecuda_context *h, const uint8_t *bytes, uint64_t byte_count,
                                               int32_t database_count, hecuda_pir_database **out) {
    if (!out || database_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument / no databases");
    for (int32_t t = 0; t < database_count; ++t) out[t] = nullptr;
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null buffer");
    const Context &c = *h->ctx;
    CodecConsts cc;
    std::string err;
    if (!codec_consts(c, c.map_q(c.L), 0, cc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const long long plaintext_bytes = serialized_poly_bytes(cc);
    std::vector<long long> tag;
    const dbio::TagWalk walk = dbio::walk_tags(bytes, (long long)std::min<uint64_t>(byte_count, INT64_MAX), plaintext_bytes, tag);
    if (walk.error != dbio::TagWalk::kOk) return load_refusal(walk, byte_count, plaintext_bytes);
    if (walk.count == 0) return fail(HECUDA_ERR_INVALID_ARGUMENT, "emptyDatabase: no plaintexts to load");
    if (walk.count % database_count)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "invalidDatabasePlaintextCount(plaintextCount: " + std::to_string(walk.count) +
                                                     ", expected: a multiple of " + std::to_string(database_count) + ")");
    const int64_t per_db = walk.count / database_count;
    long long widest = 0;
    const std::vector<DbChunk> plan = plan_db_chunks(tag, std::vector<int64_t>((size_t)database_count, per_db), widest);
    const bool pinned = host_pinned(bytes, (size_t)tag.back());
    const bool narrow = inner_product_plain_small_supported(c, c.L);
    const size_t rows_words = (size_t)c.L * c.n * per_db;

    DbStaging st(h);
    if (!st.g0.w || !st.g1.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const cudaStream_t *streams = st.stream;
    std::vector<hecuda_pir_database *> dbs;
    long long *d_tag = nullptr;
    unsigned long long *d_bad = nullptr, bad = ~0ull;
    cudaError_t e = cudaSuccess;
    for (int32_t t = 0; t < database_count && e == cudaSuccess; ++t) {
        hecuda_pir_database *db = new (std::nothrow) hecuda_pir_database();
        if (!db) {
            e = cudaErrorMemoryAllocation;
            break;
        }
        db->owner = h;
        db->count = per_db;
        dbs.push_back(db);
        e = narrow ? cudaMalloc(&db->d_plain32, rows_words * sizeof(u32)) : cudaMalloc(&db->d_plain, rows_words * sizeof(u64));
        if (e == cudaSuccess) e = cudaMalloc(&db->d_present, (size_t)per_db);
    }
    if (e == cudaSuccess) e = cudaMalloc(&d_tag, tag.size() * sizeof(long long));
    if (e == cudaSuccess) e = upload(d_tag, tag.data(), tag.size() * sizeof(long long));
    if (e == cudaSuccess) e = cudaMalloc(&d_bad, sizeof(unsigned long long));
    if (e == cudaSuccess) e = fill(d_bad, 0xff, sizeof(unsigned long long));
    if (e == cudaSuccess) e = st.init((size_t)widest, !pinned);
    for (size_t k = 0; k < plan.size() && e == cudaSuccess; ++k) {
        const int b = (int)(k & 1);
        const dbio::Chunk &ch = plan[k].chunk;
        const long long base = tag[(size_t)ch.first], size = tag[(size_t)(ch.first + ch.count)] - base;
        const unsigned char *src = bytes + base;
        if (!pinned) {  // the pinned buffer is free once the copy two chunks back has finished
            if (k >= 2) e = cudaEventSynchronize(st.copied[b]);
            if (e != cudaSuccess) break;
            memcpy(st.host[b], src, (size_t)size);
            src = st.host[b];
        }
        e = cudaMemcpyAsync(st.dev[b], src, (size_t)size, cudaMemcpyHostToDevice, streams[b]);
        if (e == cudaSuccess && !pinned) e = cudaEventRecord(st.copied[b], streams[b]);
        hecuda_pir_database *db = dbs[(size_t)plan[k].db];
        const PolyLayout at{d_tag, base, ch.first, db->d_present + plan[k].local, d_bad};
        if (e == cudaSuccess)
            e = resident_rows(c, db).with(plan[k].local, [&](auto *rows) {
                return launch_poly_load(c, cc, 0, st.dev[b], rows, ch.count, streams[b], at);
            });
    }
    for (int b = 0; b < 2; ++b) {
        const cudaError_t e2 = cudaStreamSynchronize(streams[b]);
        if (e == cudaSuccess) e = e2;
    }
    if (e == cudaSuccess) e = cudaMemcpy(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost);
    cudaFree(d_tag);
    cudaFree(d_bad);
    if (e == cudaSuccess && bad == ~0ull) {
        for (int32_t t = 0; t < database_count; ++t) out[t] = dbs[(size_t)t];
        return HECUDA_OK;
    }
    for (hecuda_pir_database *db : dbs) hecuda_pir_database_destroy(db);
    if (e != cudaSuccess) return cuda_fail(e, "pir databases from serialized bytes");
    const int row = (int)(bad % (unsigned long long)c.L);
    return fail(HECUDA_ERR_INVALID_ARGUMENT, corrupted("plaintext " + std::to_string(bad / (unsigned long long)c.L) + ", row " +
                                                       std::to_string(row) + ": a residue is not below q_" + std::to_string(row) +
                                                       " = " + std::to_string(cc.modulus[row])));
}

int32_t hecuda_pir_databases_serialized_byte_count(const hecuda_pir_database *const *dbs, int32_t database_count,
                                                   uint64_t *bytes) {
    if (!bytes) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    CodecConsts cc;
    std::vector<long long> tag;
    int32_t rc = serialization_plan(dbs, database_count, cc, tag);
    if (rc) return rc;
    *bytes = (uint64_t)tag.back();
    return HECUDA_OK;
}

int32_t hecuda_pir_databases_serialize(const hecuda_pir_database *const *dbs, int32_t database_count, uint8_t *out,
                                       uint64_t capacity, uint64_t *written) {
    if (!out || !written) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    *written = 0;
    CodecConsts cc;
    std::vector<long long> tag;
    int32_t rc = serialization_plan(dbs, database_count, cc, tag);
    if (rc) return rc;
    const uint64_t size = (uint64_t)tag.back();
    if (capacity < size)
        return fail(HECUDA_ERR_INVALID_ARGUMENT, "capacity " + std::to_string(capacity) + " below the serialized size " +
                                                     std::to_string(size));
    const hecuda_context *h = dbs[0]->owner;
    const Context &c = *h->ctx;
    const long long count = (long long)tag.size() - 1;
    out[0] = (uint8_t)dbio::kVersion;
    for (int k = 0; k < 4; ++k) out[1 + k] = (uint8_t)(count >> (8 * k));
    std::vector<int64_t> counts((size_t)database_count);
    for (int32_t t = 0; t < database_count; ++t) counts[(size_t)t] = dbs[t]->count;
    long long widest = 0;
    const std::vector<DbChunk> plan = plan_db_chunks(tag, counts, widest);
    const bool pinned = host_pinned(out, (size_t)size);
    DbStaging st(h);
    if (!st.g0.w || !st.g1.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const cudaStream_t *streams = st.stream;
    long long *d_tag = nullptr;
    cudaError_t e = cudaMalloc(&d_tag, tag.size() * sizeof(long long));
    if (e == cudaSuccess) e = upload(d_tag, tag.data(), tag.size() * sizeof(long long));
    if (e == cudaSuccess) e = st.init((size_t)widest, !pinned);
    // a pageable `out`: chunk k's pinned bytes are copied out once chunk k + 1 is enqueued
    auto drain = [&](size_t k) {
        const dbio::Chunk &ch = plan[k].chunk;
        const long long base = tag[(size_t)ch.first];
        cudaError_t e2 = cudaEventSynchronize(st.copied[k & 1]);
        if (e2 == cudaSuccess) memcpy(out + base, st.host[k & 1], (size_t)(tag[(size_t)(ch.first + ch.count)] - base));
        return e2;
    };
    for (size_t k = 0; k < plan.size() && e == cudaSuccess; ++k) {
        const int b = (int)(k & 1);
        const dbio::Chunk &ch = plan[k].chunk;
        const long long base = tag[(size_t)ch.first], bytes = tag[(size_t)(ch.first + ch.count)] - base;
        const PolyLayout at{d_tag, base, ch.first, nullptr, nullptr};
        e = resident_rows(c, dbs[plan[k].db]).with(plan[k].local, [&](const auto *rows) {
            return launch_poly_serialize(c, cc, 0, rows, st.dev[b], ch.count, streams[b], at);
        });
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(pinned ? out + base : st.host[b], st.dev[b], (size_t)bytes, cudaMemcpyDeviceToHost, streams[b]);
        if (e == cudaSuccess && !pinned) e = cudaEventRecord(st.copied[b], streams[b]);
        if (e == cudaSuccess && !pinned && k >= 1) e = drain(k - 1);
    }
    if (e == cudaSuccess && !pinned && !plan.empty()) e = drain(plan.size() - 1);
    for (int b = 0; b < 2; ++b) {
        const cudaError_t e2 = cudaStreamSynchronize(streams[b]);
        if (e == cudaSuccess) e = e2;
    }
    cudaFree(d_tag);
    if (e != cudaSuccess) return cuda_fail(e, "pir databases serialize");
    *written = size;
    return HECUDA_OK;
}

int32_t hecuda_mulpir_expand_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *cts, int32_t ct_count,
                                    int64_t output_count, uint64_t *out, void *stream) {
    int32_t rc = check_expand_args(h, k, cts, ct_count, output_count, out);
    if (rc) return rc;
    return expand_device(h, &k, 1, (const u64 *)cts, ct_count, output_count, (u64 *)out, (cudaStream_t)stream);
}

int32_t hecuda_mulpir_expand(const hecuda_context *h, const hecuda_evk *k, const uint64_t *cts, int32_t ct_count,
                             int64_t output_count, uint64_t *out) {
    int32_t rc = check_expand_args(h, k, cts, ct_count, output_count, out);
    if (rc) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const size_t ct_words = (size_t)2 * h->ctx->L * h->ctx->n;
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    u64 *d_in = nullptr, *d_out = nullptr;
    CK(tmp.alloc(&d_in, ct_words * ct_count));
    CK(tmp.alloc(&d_out, ct_words * output_count));
    DrainOnExit drain{s};  // copies of the caller's buffers are in flight on `s` from here on
    CK(cudaMemcpyAsync(d_in, cts, ct_words * ct_count * sizeof(u64), cudaMemcpyHostToDevice, s));
    if ((rc = expand_device(h, &k, 1, d_in, ct_count, output_count, d_out, s))) return rc;
    CK(cudaMemcpyAsync(out, d_out, ct_words * output_count * sizeof(u64), cudaMemcpyDeviceToHost, s));
    CK(wait_stream(s));
    return HECUDA_OK;
}

int32_t hecuda_mulpir_compute_response_device(const hecuda_context *h, const hecuda_evk *k,
                                              const hecuda_pir_database *const *dbs, int32_t db_count, const int32_t *dims,
                                              int32_t dim_count, int32_t chunk_count, const uint64_t *query,
                                              int32_t query_ct_count, int32_t indices_count, uint64_t *out, void *stream) {
    ResponseShape shape;
    int32_t rc = check_response_args(h, k, dbs, db_count, dims, dim_count, chunk_count, query, query_ct_count,
                                     indices_count, out, shape);
    if (rc) return rc;
    return respond_group(h, &k, 1, -1, dbs, db_count, shape, (const u64 *)query, query_ct_count, indices_count, (u64 *)out,
                         (cudaStream_t)stream);
}

int32_t hecuda_mulpir_compute_response(const hecuda_context *h, const hecuda_evk *k, const hecuda_pir_database *const *dbs,
                                       int32_t db_count, const int32_t *dims, int32_t dim_count, int32_t chunk_count,
                                       const uint64_t *query, int32_t query_ct_count, int32_t indices_count,
                                       uint64_t *out) {
    ResponseShape shape;
    int32_t rc = check_response_args(h, k, dbs, db_count, dims, dim_count, chunk_count, query, query_ct_count,
                                     indices_count, out, shape);
    if (rc) return rc;
    if (indices_count == 1 && db_count == 1) {  // replay the captured pipeline of this (database, key, shape)
        WsGuard g(h);
        if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
        cudaStream_t s = g.w->stream;
        PirGraph *pg = acquire_graph(h, k, dbs[0], shape, query_ct_count, s, &rc);
        if (rc) return rc;
        if (pg) {
            const Context &c = *h->ctx;
            cudaError_t e = cudaMemcpyAsync(pg->d_query, query, (size_t)2 * c.L * c.n * query_ct_count * sizeof(u64),
                                            cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaGraphLaunch(pg->exec, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(out, pg->d_out, (size_t)2 * c.n * chunk_count * sizeof(u64), cudaMemcpyDeviceToHost, s);
            // on every path: the instance and the caller's buffers are only free once `s` has drained
            const cudaError_t drained = wait_stream(s);
            if (e == cudaSuccess) e = drained;
            g_kernel_launches += pg->launches;
            release_graph(h, pg);
            if (e != cudaSuccess) return cuda_fail(e, "response graph");
            return HECUDA_OK;
        }
    }  // not capturable on this setup, or several indices / databases: the direct path
    return respond_words(h, &k, 1, true, dbs, db_count, shape, query, query_ct_count, indices_count, out);
}

int32_t hecuda_mulpir_compute_response_clients_device(const hecuda_context *h, const hecuda_evk *const *evks,
                                                      int32_t client_count, const hecuda_pir_database *const *dbs,
                                                      int32_t db_count, const int32_t *dims, int32_t dim_count,
                                                      int32_t chunk_count, const uint64_t *queries, int32_t query_ct_count,
                                                      int32_t indices_count, uint64_t *out, void *stream) {
    ResponseShape shape;
    int32_t rc = check_clients_args(h, evks, client_count, dbs, db_count, dims, dim_count, chunk_count, queries,
                                    query_ct_count, indices_count, out, shape);
    if (rc) return rc;
    const size_t query_words = (size_t)2 * h->ctx->L * h->ctx->n * query_ct_count;
    const size_t out_words = (size_t)2 * h->ctx->n * chunk_count * indices_count;
    for (int32_t first = 0; first < client_count; first += HECUDA_MULPIR_CLIENT_GROUP) {
        const int clients = std::min<int32_t>(HECUDA_MULPIR_CLIENT_GROUP, client_count - first);
        rc = respond_group(h, evks + first, clients, first, dbs, db_count, shape, (const u64 *)queries + query_words * first,
                           query_ct_count, indices_count, (u64 *)out + out_words * first, (cudaStream_t)stream);
        if (rc) return rc;
    }
    return HECUDA_OK;
}

int32_t hecuda_mulpir_compute_response_clients(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                                               const hecuda_pir_database *const *dbs, int32_t db_count, const int32_t *dims,
                                               int32_t dim_count, int32_t chunk_count, const uint64_t *queries,
                                               int32_t query_ct_count, int32_t indices_count, uint64_t *out) {
    ResponseShape shape;
    int32_t rc = check_clients_args(h, evks, client_count, dbs, db_count, dims, dim_count, chunk_count, queries,
                                    query_ct_count, indices_count, out, shape);
    if (rc) return rc;
    return respond_words(h, evks, client_count, false, dbs, db_count, shape, queries, query_ct_count, indices_count, out);
}

int32_t hecuda_mulpir_compute_response_wire(const hecuda_context *h, const hecuda_evk *k, const hecuda_pir_database *const *dbs,
                                            int32_t db_count, const int32_t *dims, int32_t dim_count, int32_t chunk_count,
                                            const uint8_t *query_poly0, const uint8_t *query_seeds, int32_t query_ct_count,
                                            int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                            uint8_t *out) {
    ResponseShape shape;
    int32_t rc = check_response_args(h, k, dbs, db_count, dims, dim_count, chunk_count, (const uint64_t *)query_poly0,
                                     query_ct_count, indices_count, out, shape);
    if (rc) return rc;
    return respond_wire(h, &k, 1, true, dbs, db_count, shape, query_poly0, query_seeds, query_ct_count, indices_count,
                        skip_lsbs_poly0, skip_lsbs_poly1, out);
}

int32_t hecuda_mulpir_compute_response_clients_wire(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                                                    const hecuda_pir_database *const *dbs, int32_t db_count, const int32_t *dims,
                                                    int32_t dim_count, int32_t chunk_count, const uint8_t *query_poly0,
                                                    const uint8_t *query_seeds, int32_t query_ct_count, int32_t indices_count,
                                                    int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1, uint8_t *out) {
    ResponseShape shape;
    int32_t rc = check_clients_args(h, evks, client_count, dbs, db_count, dims, dim_count, chunk_count,
                                    (const uint64_t *)query_poly0, query_ct_count, indices_count, out, shape);
    if (rc) return rc;
    return respond_wire(h, evks, client_count, false, dbs, db_count, shape, query_poly0, query_seeds, query_ct_count,
                        indices_count, skip_lsbs_poly0, skip_lsbs_poly1, out);
}

// The walk of every client's EncryptedIndices, checked like hecuda_mulpir_compute_response_clients_wire's arguments
int32_t hecuda_mulpir_compute_response_clients_proto(const hecuda_context *h, const hecuda_evk *const *evks, int32_t client_count,
                                                     const hecuda_pir_database *const *dbs, int32_t db_count,
                                                     const int32_t *dims, int32_t dim_count, int32_t chunk_count,
                                                     const uint8_t *const *messages, const uint64_t *message_byte_counts,
                                                     int32_t indices_count, int32_t skip_lsbs_poly0, int32_t skip_lsbs_poly1,
                                                     uint8_t *out) {
    int32_t rc = check_ctx(h);
    if (rc) return rc;
    if (!messages || !message_byte_counts || !dims || dim_count < 1) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *h->ctx;
    int64_t expanded = 0;
    for (int32_t d = 0; d < dim_count; ++d) expanded += dims[d];
    // the ciphertext count of the parameter's query (MulPirClient.generateQuery: expandedQueryCount x indicesCount
    // compressed into ciphertexts of N coefficients)
    const int64_t query_ct_count = indices_count > 0 && expanded > 0 ? (expanded * indices_count + c.n - 1) / c.n : 1;
    if (query_ct_count > 0x7fffffff) return fail(HECUDA_ERR_UNSUPPORTED, "too many query ciphertexts");
    ResponseShape shape;
    if ((rc = check_clients_args(h, evks, client_count, dbs, db_count, dims, dim_count, chunk_count,
                                 (const uint64_t *)messages, (int32_t)query_ct_count, indices_count, out, shape)))
        return rc;
    uint64_t size = 0;
    if ((rc = hecuda_mulpir_response_proto_byte_count(h, chunk_count, indices_count, skip_lsbs_poly0, skip_lsbs_poly1, &size)))
        return rc;
    CodecConsts qc;
    std::string err;
    if (!codec_consts(c, c.map_q(c.L), 0, qc, err)) return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    const pirproto::PolySizes sz = pirproto::poly_sizes(qc, c.n);
    std::vector<pirproto::Query> queries((size_t)client_count);
    for (int32_t j = 0; j < client_count; ++j) {
        const std::string who = "client " + std::to_string(j) + ": ";
        if (!messages[j]) return fail(HECUDA_ERR_INVALID_ARGUMENT, who + "null argument");
        pirproto::Error e;
        if (!pirproto::walk_encrypted_indices(messages[j], 0, (long long)message_byte_counts[j], sz, queries[(size_t)j], e))
            return fail(e.code, who + e.what);
        if (!pirproto::check_query(queries[(size_t)j], (uint64_t)indices_count, (size_t)query_ct_count, e))
            return fail(e.code, who + e.what);
    }
    WireCodec wc;
    if ((rc = wc.setup(c, skip_lsbs_poly0, skip_lsbs_poly1))) return rc;
    const pirproto::ResponseLayout layout = pirproto::place_response(indices_count, chunk_count, (long long)wc.bytes[0],
                                                                     (long long)wc.bytes[1], skip_lsbs_poly0, skip_lsbs_poly1);
    return respond_proto(h, evks, client_count, dbs, db_count, shape, messages, message_byte_counts, queries,
                         (int32_t)query_ct_count, indices_count, skip_lsbs_poly0, skip_lsbs_poly1, layout, out);
}

}  // extern "C"
