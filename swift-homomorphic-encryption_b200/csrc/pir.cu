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
// Everything is enqueued on one stream; concurrent queries (different clients, different keys) run on different
// streams from different host threads.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include <set>

#include "capi_internal.hpp"

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

struct RowConsts {
    int rows;
    u64 p[kMaxRows];
};

// one node of an expansion level: where its two children go
struct ExpandStep {
    int dst0, dst1;
    unsigned flags;  // 1: p0 is a leaf (goes to `out`), 2: p0 doubled, 4: p1 is a leaf, 8: p1 doubled
};

__device__ __forceinline__ u64 add_mod(u64 a, u64 b, u64 p) {
    const u64 s = a + b;
    return s >= p ? s - p : s;
}

// expandCiphertextForOneStep after the Galois step (PirUtil.swift:230-235) for every node of a level:
//   p0 = c1 + ct,  p1 = multiplyPowerOfX(ct - c1, -2^(logStep-1))   [gather form of PolyRq.swift:398-422]
__global__ void __launch_bounds__(256) expand_combine_kernel(const u64 *__restrict__ cur, const u64 *__restrict__ c1,
                                                            u64 *__restrict__ next, u64 *__restrict__ out,
                                                            const ExpandStep *__restrict__ steps,
                                                            const __grid_constant__ RowConsts c, int logn, unsigned s) {
    const int n = 1 << logn;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int pr = blockIdx.y;  // poly * rows + row
    const u64 p = c.p[pr % c.rows];
    const int64_t ct_words = (int64_t)2 * c.rows * n;
    const int64_t base = (int64_t)blockIdx.z * ct_words + (int64_t)pr * n;
    const ExpandStep st = steps[blockIdx.z];
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

RowConsts row_consts(const Context &c, int l) {
    RowConsts rc;
    const NttRowMap map = c.map_q(l);
    rc.rows = l;
    for (int r = 0; r < l; ++r) rc.p[r] = c.slots[map.slot[r]].dev.p;
    return rc;
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

// PirUtil.expand on device buffers: d_in = ct_count canonical (Coeff) ciphertexts of L rows, d_out = output_count
// d_steps_ready: the plan's steps already on the device (captured graphs upload them once, outside the capture)
int32_t expand_device(const hecuda_context *h, const hecuda_evk *k, const u64 *d_in, int64_t ct_count, int64_t output_count,
                      u64 *d_out, cudaStream_t s, const void *d_steps_ready = nullptr) {
    const Context &c = *h->ctx;
    const int l = c.L;
    const int64_t n = c.n;
    const size_t ct_words = (size_t)2 * l * n;
    const ExpandPlan plan = build_expand_plan(n, ct_count, output_count);
    for (const auto &leaf : plan.root_leaves)
        CK(cudaMemcpyAsync(d_out + ct_words * leaf.second, d_in + ct_words * leaf.first, ct_words * sizeof(u64),
                           cudaMemcpyDeviceToDevice, s));
    if (plan.levels.empty()) return HECUDA_OK;
    StreamBuffers tmp(s);
    u64 *level_buf[2] = {nullptr, nullptr}, *c1_buf[2] = {nullptr, nullptr}, *scratch = nullptr;
    ExpandStep *d_steps = nullptr;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(h->chunk, plan.max_nodes));
    CK(tmp.alloc(&level_buf[0], ct_words * plan.max_nodes));
    CK(tmp.alloc(&level_buf[1], ct_words * plan.max_nodes));
    CK(tmp.alloc(&c1_buf[0], ct_words * plan.max_nodes));
    CK(tmp.alloc(&c1_buf[1], ct_words * plan.max_nodes));
    CK(tmp.alloc(&scratch, galois_scratch_words(c, l) * (size_t)chunk));
    if (d_steps_ready) {
        d_steps = (ExpandStep *)d_steps_ready;
    } else {
        CK(tmp.alloc_bytes((void **)&d_steps, plan.steps.size() * sizeof(ExpandStep)));
        CK(cudaMemcpyAsync(d_steps, plan.steps.data(), plan.steps.size() * sizeof(ExpandStep), cudaMemcpyHostToDevice, s));
        CK(wait_stream(s));  // plan.steps is a pageable temporary
    }
    const RowConsts rc = row_consts(c, l);
    const int threads = n >= 256 ? 256 : (n < 32 ? 32 : (int)n);
    const u64 *cur = d_in;  // the active roots are a prefix of the input (only the last one can be a single output)
    int flip = 0;
    for (const PlanLevel &level : plan.levels) {
        unsigned element = 0;
        int times = 0;
        const u64 *key = nullptr;
        int32_t rc32 = pick_galois(k, n, level.log_step, &element, &times, &key);
        if (rc32) return rc32;
        const u64 *c1 = cur;
        for (int t = 0; t < times; ++t) {  // c1.applyGalois(element:using:) `times` times (:223-227)
            u64 *dst = c1_buf[t & 1];
            for (int64_t done = 0; done < level.nodes; done += chunk) {
                const int64_t items = std::min<int64_t>(chunk, level.nodes - done);
                cudaError_t e = apply_galois_chunk(c, scratch, key, c1 + ct_words * done, l, element, dst + ct_words * done,
                                                   items, s);
                if (e != cudaSuccess) return cuda_fail(e, "expand: applyGalois");
            }
            c1 = dst;
        }
        u64 *next = level_buf[flip];
        flip ^= 1;
        const unsigned shift = (unsigned)(2 * n) - (1u << (level.log_step - 1));  // -2^(logStep-1) mod 2N
        for (int64_t done = 0; done < level.nodes;) {
            const int64_t items = std::min<int64_t>(level.nodes - done, 65535);
            dim3 grid((unsigned)((n + threads - 1) / threads), (unsigned)(2 * l), (unsigned)items);
            ++g_kernel_launches;
            expand_combine_kernel<<<grid, threads, 0, s>>>(cur + ct_words * done, c1 + ct_words * done, next, d_out,
                                                           d_steps + level.step_offset + done, rc, c.logn, shift);
            done += items;
        }
        CK(cudaGetLastError());
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

// PirUtil.computeResponse (PirUtil.swift:490-568) for device-resident query ciphertexts; d_out receives
// indices_count x chunk_count ciphertexts of 2 x 1 x N (Coeff, one modulus)
int32_t compute_response_device(const hecuda_context *h, const hecuda_evk *k, const hecuda_pir_database *const *dbs,
                                int32_t db_count, const ResponseShape &shape, const u64 *d_query, int64_t query_ct_count,
                                int64_t indices_count, u64 *d_out, cudaStream_t s, const void *d_steps_ready = nullptr) {
    const Context &c = *h->ctx;
    const int L = c.L;
    const int64_t n = c.n;
    const size_t ct_words = (size_t)2 * L * n;
    const int64_t eqc = shape.expanded_query_count, dim0 = shape.dims[0];
    const int64_t rows = shape.chunk_count * shape.columns;  // first-dimension inner products per query
    StreamBuffers tmp(s);
    u64 *expanded = nullptr, *first_eval = nullptr, *results[2] = {nullptr, nullptr}, *lhs = nullptr, *ct3 = nullptr,
        *scratch = nullptr;
    CK(tmp.alloc(&expanded, ct_words * eqc * indices_count));
    int32_t rc = expand_device(h, k, d_query, query_ct_count, eqc * indices_count, expanded, s, d_steps_ready);
    if (rc) return rc;
    CK(tmp.alloc(&first_eval, ct_words * dim0));
    CK(tmp.alloc(&results[0], ct_words * rows));
    CK(tmp.alloc(&results[1], ct_words * rows));
    size_t scratch_words = 0, lhs_words = 0, ct3_words = 0;
    {
        int64_t count = rows;
        for (size_t d = 1; d < shape.dims.size(); ++d) {
            const int64_t size = shape.dims[d], groups = count / size;
            scratch_words = std::max(scratch_words, inner_product_scratch_words(c, size) * (size_t)groups);
            scratch_words = std::max(scratch_words, relinearize_scratch_words(c, L) * (size_t)groups);
            lhs_words = std::max(lhs_words, ct_words * (size_t)(size * groups));
            ct3_words = std::max(ct3_words, (size_t)3 * L * n * groups);
            count = groups;
        }
    }
    CK(tmp.alloc(&scratch, scratch_words));
    CK(tmp.alloc(&lhs, lhs_words));
    CK(tmp.alloc(&ct3, ct3_words));
    const NttRowMap map = c.map_q(L);
    for (int64_t qi = 0; qi < indices_count; ++qi) {
        const u64 *cts = expanded + ct_words * eqc * qi;
        const hecuda_pir_database *db = dbs[db_count == 1 ? 0 : qi];
        cudaError_t e;
        // firstDimensionQueries: convertToEvalFormat (:523-532)
        if ((e = launch_ntt_forward(c, map, cts, first_eval, dim0 * 2 * L, s)) != cudaSuccess) return cuda_fail(e, "ntt");
        // every column of every chunk: Scheme.innerProduct(ciphertexts:plaintexts:) then convertToCanonicalFormat (:427-435)
        e = db->d_plain32 ? launch_inner_product_plain_small(c, first_eval, 2, L, dim0, db->d_plain32, db->d_present, results[0], rows, s)
                          : launch_inner_product_plain(c, first_eval, 2, L, dim0, db->d_plain, db->d_present, results[0], rows, s);
        if (e != cudaSuccess)
            return cuda_fail(e, "innerProduct(ciphertexts:plaintexts:)");
        if ((e = launch_ntt_inverse(c, map, results[0], results[0], rows * 2 * L, kScalePlain, s)) != cudaSuccess)
            return cuda_fail(e, "ntt");
        int64_t count = rows, query_start = dim0;
        int cur = 0;
        for (size_t d = 1; d < shape.dims.size(); ++d) {  // remaining dimensions (:447-480)
            const int64_t size = shape.dims[d], groups = count / size;
            for (int64_t g = 0; g < groups; ++g)  // vector0 = the same query slice for every group
                CK(cudaMemcpyAsync(lhs + ct_words * size * g, cts + ct_words * query_start, ct_words * size * sizeof(u64),
                                   cudaMemcpyDeviceToDevice, s));
            if ((e = inner_product_chunk(c, scratch, lhs, results[cur], size, ct3, groups, s)) != cudaSuccess)
                return cuda_fail(e, "innerProduct");
            if ((e = relinearize_chunk(c, scratch, k->d_relin, ct3, L, results[cur ^ 1], groups, s)) != cudaSuccess)
                return cuda_fail(e, "relinearize");
            cur ^= 1;
            count = groups;
            query_start += size;
        }
        if (count != shape.chunk_count)
            return fail(HECUDA_ERR_INVALID_ARGUMENT, "There should be only 1 ciphertext in the final result for each chunk");
        // modSwitchDownToSingle (HeScheme.swift:1481-1485); BFV's canonical format is already Coeff
        u64 *final_out = d_out + (size_t)2 * n * shape.chunk_count * qi;
        if (L == 1) {
            CK(cudaMemcpyAsync(final_out, results[cur], (size_t)2 * n * count * sizeof(u64), cudaMemcpyDeviceToDevice, s));
        }
        for (int l = L; l > 1; --l) {
            u64 *dst = l == 2 ? final_out : results[cur ^ 1];
            if ((e = launch_mod_switch(c, results[cur], l, dst, count * 2, s)) != cudaSuccess) return cuda_fail(e, "modSwitchDown");
            cur ^= 1;
        }
    }
    return HECUDA_OK;
}

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
    void *d_steps = nullptr;
    unsigned long long launches = 0;  // kernels inside the graph (for hecuda_kernel_launch_count)
    bool busy = false;
    void release() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        if (d_query) cudaFree(d_query);
        if (d_out) cudaFree(d_out);
        if (d_steps) cudaFree(d_steps);
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
    const size_t ct_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * c.n * shape.chunk_count;
    PirGraph *g = new (std::nothrow) PirGraph();
    if (!g) return nullptr;
    g->evk = k;
    g->evk_version = k->version;
    g->db = db;
    g->dims = shape.dims;
    g->chunk_count = shape.chunk_count;
    g->query_ct_count = query_ct_count;
    const ExpandPlan plan = build_expand_plan(c.n, query_ct_count, shape.expanded_query_count);
    cudaError_t e = cudaMalloc(&g->d_query, ct_words * query_ct_count * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&g->d_out, out_words * sizeof(u64));
    if (e == cudaSuccess) e = cudaMalloc(&g->d_steps, std::max<size_t>(plan.steps.size(), 1) * sizeof(ExpandStep));
    if (e == cudaSuccess && !plan.steps.empty()) e = upload(g->d_steps, plan.steps.data(), plan.steps.size() * sizeof(ExpandStep));
    if (e != cudaSuccess) {
        g->release();
        delete g;
        *rc = cuda_fail(e, "response graph buffers");
        return nullptr;
    }
    e = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
    int32_t body = HECUDA_OK;
    if (e == cudaSuccess) {
        const hecuda_pir_database *dbs[1] = {db};
        body = compute_response_device(hc, k, dbs, 1, shape, g->d_query, query_ct_count, 1, g->d_out, s, g->d_steps);
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

}  // namespace

extern "C" {

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
            const int64_t slab = std::max<int64_t>(1, (int64_t)((size_t)8 * 1024 * 1024 / c.n));
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
    if (e == cudaSuccess && inner_product_plain_small_supported(c, c.L)) {
        // small moduli (the default PIR parameters): keep the rows as uint32 -- half the bytes per scan, half the HBM
        e = cudaMalloc(&db->d_plain32, row_words * count * sizeof(u32));
        if (e == cudaSuccess) e = launch_narrow(db->d_plain, db->d_plain32, (int64_t)(row_words * count), nullptr);
        if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
        if (e == cudaSuccess) {
            cudaFree(db->d_plain);
            db->d_plain = nullptr;
        }
    }
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

int32_t hecuda_mulpir_expand_device(const hecuda_context *h, const hecuda_evk *k, const uint64_t *cts, int32_t ct_count,
                                    int64_t output_count, uint64_t *out, void *stream) {
    int32_t rc = check_expand_args(h, k, cts, ct_count, output_count, out);
    if (rc) return rc;
    return expand_device(h, k, (const u64 *)cts, ct_count, output_count, (u64 *)out, (cudaStream_t)stream);
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
    CK(cudaMemcpyAsync(d_in, cts, ct_words * ct_count * sizeof(u64), cudaMemcpyHostToDevice, s));
    rc = expand_device(h, k, d_in, ct_count, output_count, d_out, s);
    if (rc) {
        wait_stream(s);
        return rc;
    }
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
    return compute_response_device(h, k, dbs, db_count, shape, (const u64 *)query, query_ct_count, indices_count,
                                   (u64 *)out, (cudaStream_t)stream);
}

int32_t hecuda_mulpir_compute_response(const hecuda_context *h, const hecuda_evk *k, const hecuda_pir_database *const *dbs,
                                       int32_t db_count, const int32_t *dims, int32_t dim_count, int32_t chunk_count,
                                       const uint64_t *query, int32_t query_ct_count, int32_t indices_count,
                                       uint64_t *out) {
    ResponseShape shape;
    int32_t rc = check_response_args(h, k, dbs, db_count, dims, dim_count, chunk_count, query, query_ct_count,
                                     indices_count, out, shape);
    if (rc) return rc;
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    const Context &c = *h->ctx;
    const size_t ct_words = (size_t)2 * c.L * c.n, out_words = (size_t)2 * c.n * chunk_count * indices_count;
    cudaStream_t s = g.w->stream;
    if (indices_count == 1 && db_count == 1) {
        PirGraph *pg = acquire_graph(h, k, dbs[0], shape, query_ct_count, s, &rc);
        if (rc) return rc;
        if (pg) {
            cudaError_t e = cudaMemcpyAsync(pg->d_query, query, ct_words * query_ct_count * sizeof(u64), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaGraphLaunch(pg->exec, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(out, pg->d_out, out_words * sizeof(u64), cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = wait_stream(s);
            g_kernel_launches += pg->launches;
            release_graph(h, pg);
            if (e != cudaSuccess) return cuda_fail(e, "response graph");
            return HECUDA_OK;
        }
    }
    StreamBuffers tmp(s);
    u64 *d_query = nullptr, *d_out = nullptr;
    CK(tmp.alloc(&d_query, ct_words * query_ct_count));
    CK(tmp.alloc(&d_out, out_words));
    CK(cudaMemcpyAsync(d_query, query, ct_words * query_ct_count * sizeof(u64), cudaMemcpyHostToDevice, s));
    rc = compute_response_device(h, k, dbs, db_count, shape, d_query, query_ct_count, indices_count, d_out, s);
    if (rc) {
        wait_stream(s);
        return rc;
    }
    CK(cudaMemcpyAsync(out, d_out, out_words * sizeof(u64), cudaMemcpyDeviceToHost, s));
    CK(wait_stream(s));
    return HECUDA_OK;
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
    if (!query_seeds) return fail(HECUDA_ERR_INVALID_ARGUMENT, "null argument");
    const Context &c = *h->ctx;
    CodecConsts in_codec, out_codec[2];
    std::string err;
    if (!codec_consts(c, c.map_q(c.L), 0, in_codec, err) || !codec_consts(c, c.map_q(1), skip_lsbs_poly0, out_codec[0], err) ||
        !codec_consts(c, c.map_q(1), skip_lsbs_poly1, out_codec[1], err))
        return fail(HECUDA_ERR_INVALID_ARGUMENT, err);
    WsGuard g(h);
    if (!g.w) return fail(HECUDA_ERR_CUDA, "could not create a CUDA stream / workspace");
    cudaStream_t s = g.w->stream;
    StreamBuffers tmp(s);
    const size_t ct_words = (size_t)2 * c.L * c.n, in_bytes = (size_t)serialized_poly_bytes(in_codec);
    const int64_t replies = (int64_t)indices_count * chunk_count;
    const size_t b0 = (size_t)serialized_poly_bytes(out_codec[0]), b1 = (size_t)serialized_poly_bytes(out_codec[1]);
    unsigned char *d_poly0 = nullptr, *d_seeds = nullptr, *d_bytes[2] = {nullptr, nullptr}, *d_reply = nullptr;
    u64 *d_query = nullptr, *d_resp = nullptr, *d_polys = nullptr;
    CK(tmp.alloc_bytes((void **)&d_poly0, in_bytes * query_ct_count));
    CK(tmp.alloc_bytes((void **)&d_seeds, (size_t)32 * query_ct_count));
    CK(tmp.alloc(&d_query, ct_words * query_ct_count));
    CK(tmp.alloc(&d_resp, (size_t)2 * c.n * replies));
    CK(tmp.alloc(&d_polys, (size_t)2 * c.n * replies));
    CK(tmp.alloc_bytes((void **)&d_bytes[0], ((b0 + 7) & ~(size_t)7) * replies + 8));
    CK(tmp.alloc_bytes((void **)&d_bytes[1], ((b1 + 7) & ~(size_t)7) * replies + 8));
    CK(tmp.alloc_bytes((void **)&d_reply, (b0 + b1) * replies));
    // from here on copies of the caller's buffers are in flight on `s`: every return path waits for the stream first
    struct DrainOnExit {
        cudaStream_t s;
        ~DrainOnExit() { wait_stream(s); }
    } drain{s};
    CK(cudaMemcpyAsync(d_poly0, query_poly0, in_bytes * query_ct_count, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_seeds, query_seeds, (size_t)32 * query_ct_count, cudaMemcpyHostToDevice, s));
    // Query.ciphertexts arrive as SerializedCiphertext.seeded (SerializedCiphertext.swift:41-49)
    cudaError_t e = expand_seeded_device(c, c.L, d_poly0, d_seeds, d_query, query_ct_count, s);
    if (e != cudaSuccess) return cuda_fail(e, "expand seeded query");
    rc = compute_response_device(h, k, dbs, db_count, shape, d_query, query_ct_count, indices_count, d_resp, s);
    if (rc) return rc;
    // Response ciphertexts leave as .full(polys:skipLSBs:) with Bfv.skipLSBsForDecryption (Bfv+Decrypt.swift:51-110):
    // poly 0 and poly 1 are packed with different numbers of dropped low bits
    const size_t pw = (size_t)c.n * sizeof(u64);
    for (int p = 0; p < 2; ++p) {
        const size_t bytes = p ? b1 : b0;
        CK(cudaMemcpy2DAsync(d_polys + (size_t)p * c.n * replies, pw, d_resp + (size_t)p * c.n, 2 * pw, pw, (size_t)replies,
                             cudaMemcpyDeviceToDevice, s));
        if ((e = launch_poly_serialize(c, out_codec[p], p ? skip_lsbs_poly1 : skip_lsbs_poly0, d_polys + (size_t)p * c.n * replies,
                                       d_bytes[p], replies, s)) != cudaSuccess)
            return cuda_fail(e, "serialize response");
        CK(cudaMemcpy2DAsync(d_reply + (p ? b0 : 0), b0 + b1, d_bytes[p], bytes, bytes, (size_t)replies, cudaMemcpyDeviceToDevice, s));
    }
    CK(cudaMemcpyAsync(out, d_reply, (b0 + b1) * replies, cudaMemcpyDeviceToHost, s));
    CK(wait_stream(s));
    return HECUDA_OK;
}

}  // extern "C"
