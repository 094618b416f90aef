// hybrid.cu -- hybrid search (hybrid_search / batch_hybrid_search, src/api/vectordb/search/repo.rs:168-555): reciprocal-rank
// fusion of two ranked lists per query, and the composed search that runs two of the dense, sparse and TF-IDF searches and
// fuses their results on the device.  The contract is the header comment of cdb_rrf_fuse (DESIGN.md section 8e).
// check_fuse_args and fuse_launch also serve a shard group's hybrid search (shard_group.cu, DESIGN.md section 8h).  A mixed
// batch (each query names its own pair, DESIGN.md section 8i) searches each source once and fuses each kind through row maps.
//
// rrf_fuse_kernel: one CTA per query.  Every live entry becomes (key << 32 | list << 31 | rank) in shared memory; a bitonic
// sort groups each key's entries, first list before second, each in rank order; the head of every run folds it (first
// list: the last occurrence wins; second list: or_insert then +=); the distinct keys are sorted again on
// (order_key(score) << 32 | ~key), which is f32::total_cmp descending with ties to the smaller id.  Contributions are
// recomputed from (rank, k) where they are needed, so no score array is kept.
#include <algorithm>
#include <cfloat>
#include <cstring>
#include <string>

#include "kernels.h"

namespace cdb {
namespace {

constexpr uint32_t RRF_MAX = 2048;      // entries of both lists of one query
constexpr uint32_t TF_RESULTS = 512;    // TF-IDF's bucket count: its searches return at most 512 results

// 1.0 / (rank as f32 + k + f32::EPSILON): one rounding per operation, left to right, no FMA, no approximate reciprocal
__device__ __forceinline__ float rrf_contribution(uint32_t rank, float k) {
    return __fdiv_rn(1.0f, __fadd_rn(__fadd_rn(__uint2float_rn(rank), k), FLT_EPSILON));
}

__device__ __forceinline__ uint32_t rrf_key(uint32_t id, uint32_t stride) { return stride <= 1 ? id : id - id % stride; }

// Fused row blockIdx.x reads row a.rows[i] / b.rows[i] of each list and writes row o.rows[i] (null maps: row i), so one
// launch fuses the queries of one kind of a mixed batch straight into the caller's rows.
__global__ void __launch_bounds__(1024) rrf_fuse_kernel(RrfList a, RrfList b, float k, uint32_t n_sort, uint32_t ld_out,
                                                        uint32_t *__restrict__ out_ids, float *__restrict__ out_scores,
                                                        uint32_t *__restrict__ out_counts, RrfRows o) {
    __shared__ uint64_t ent[RRF_MAX];   // (key << 32 | list << 31 | rank), ascending; ~0 = no entry
    __shared__ uint64_t res[RRF_MAX];   // (order_key(score) << 32 | ~key), descending; 0 = no key
    __shared__ uint32_t s_cnt;
    const uint32_t tid = threadIdx.x;
    const uint32_t qa = a.rows ? a.rows[blockIdx.x] : blockIdx.x, qb = b.rows ? b.rows[blockIdx.x] : blockIdx.x;
    const uint32_t q = o.rows ? o.rows[blockIdx.x] : blockIdx.x;
    const uint32_t na = min(a.counts[qa], a.ld), nb = min(b.counts[qb], b.ld), n = na + nb;
    if (tid == 0) {
        s_cnt = 0;
        if (o.err) o.err[q] = o.err_in ? o.err_in[qa] : 0;
    }
    for (uint32_t i = tid; i < n_sort; i += blockDim.x) {
        uint64_t e = ~0ull;
        if (i < na)
            e = ((uint64_t)rrf_key(a.ids[(size_t)qa * a.ld + i], a.stride) << 32) | i;
        else if (i >= a.ld && i - a.ld < nb)
            e = ((uint64_t)rrf_key(b.ids[(size_t)qb * b.ld + (i - a.ld)], b.stride) << 32) | (1u << 31) | (i - a.ld);
        ent[i] = e;
    }
    __syncthreads();
    bitonic_sort<false>(ent, n_sort);
    // a NaN k makes every contribution and every sum NaN with k's payload, quieted (x86 SSE propagation); the device's
    // own NaN results would be the canonical NaN instead
    const bool k_nan = k != k;
    const float nan_score = __uint_as_float(__float_as_uint(k) | 0x00400000u);
    for (uint32_t i = tid; i < n_sort; i += blockDim.x) {
        uint64_t r = 0;
        const uint32_t key = (uint32_t)(ent[i] >> 32);
        if (i < n && (i == 0 || (uint32_t)(ent[i - 1] >> 32) != key)) {
            float s = 0.0f;
            bool have = false;
            for (uint32_t j = i; j < n && (uint32_t)(ent[j] >> 32) == key; ++j) {
                const uint32_t lo = (uint32_t)ent[j];
                const float c = rrf_contribution(lo & 0x7FFFFFFFu, k);
                // first list: insert overwrites; second list: or_insert(c), then += c
                s = ((lo >> 31) && have) ? __fadd_rn(s, c) : c;
                have = true;
            }
            if (k_nan) s = nan_score;
            r = ((uint64_t)order_key(CDB_METRIC_DOT_PRODUCT, __float_as_uint(s)) << 32) | (uint64_t)(~key);
            atomicAdd(&s_cnt, 1u);
        }
        res[i] = r;
    }
    __syncthreads();
    bitonic_sort<true>(res, n_sort);
    const uint32_t cnt = s_cnt;
    for (uint32_t c = tid; c < ld_out; c += blockDim.x) {
        uint32_t id = CDB_INVALID_ID;
        float s = 0.0f;
        if (c < cnt) {
            id = ~(uint32_t)res[c];
            s = __uint_as_float(key_to_bits(CDB_METRIC_DOT_PRODUCT, (uint32_t)(res[c] >> 32)));
        }
        out_ids[(size_t)q * ld_out + c] = id;
        out_scores[(size_t)q * ld_out + c] = s;
    }
    if (tid == 0) out_counts[q] = cnt;
}

}  // namespace

cdb_status check_fuse_args(uint32_t ld_a, uint32_t ld_b, uint32_t nq, uint32_t ld_out, const void *ids_a, const void *cnt_a,
                           const void *ids_b, const void *cnt_b, const void *out_ids, const void *out_scores, const void *out_counts) {
    CDB_REQUIRE((uint64_t)ld_a + ld_b <= RRF_MAX, "ld_first + ld_second must be <= 2048");
    CDB_REQUIRE(ld_out >= ld_a + ld_b, "ld_out must be >= ld_first + ld_second");
    CDB_REQUIRE(!nq || (cnt_a && cnt_b && out_counts), "null counts");
    CDB_REQUIRE(!nq || ((ids_a || !ld_a) && (ids_b || !ld_b)), "null ids");
    CDB_REQUIRE(!nq || !ld_out || (out_ids && out_scores), "null output");
    return CDB_OK;
}

cdb_status fuse_launch(const RrfList &a, const RrfList &b, uint32_t nq, float k, uint32_t ld_out, uint32_t *d_ids, float *d_scores,
                       uint32_t *d_counts, cudaStream_t s, const RrfRows &o) {
    if (!nq) return CDB_OK;
    uint32_t n_sort = 2;
    while (n_sort < a.ld + b.ld) n_sort <<= 1;
    const uint32_t threads = std::min<uint32_t>(1024, std::max<uint32_t>(32, n_sort / 2));
    rrf_fuse_kernel<<<nq, threads, 0, s>>>(a, b, k, n_sort, ld_out, d_ids, d_scores, d_counts, o);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status check_kinds(const uint8_t *kinds, uint32_t nq, const uint32_t n_src[3]) {
    CDB_REQUIRE(kinds || !nq, "null kinds");
    uint32_t n[3] = {0, 0, 0};
    for (uint32_t q = 0; q < nq; ++q) {
        if (kinds[q] > CDB_HYBRID_SPARSE_TFIDF) {
            set_error("kinds[" + std::to_string(q) + "] = " + std::to_string(kinds[q]) + ": a kind is 0, 1 or 2");
            return CDB_INVALID_PARAMS;
        }
        ++n[HYB_KIND_SRC[kinds[q]][0]];
        ++n[HYB_KIND_SRC[kinds[q]][1]];
    }
    CDB_REQUIRE(n[0] == n_src[0] && n[1] == n_src[1] && n[2] == n_src[2],
                "n_dense, n_sparse and n_tfidf must be the numbers of queries whose kinds name each source");
    return CDB_OK;
}

void mixed_chunks(const uint8_t *kinds, uint32_t nq, uint32_t chunk, std::vector<MixedChunk> *chunks, std::vector<uint32_t> *maps) {
    maps->assign((size_t)3 * nq, 0);
    uint32_t next[3] = {0, 0, 0};   // each source's next row
    size_t at = 0;
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
        MixedChunk c{};
        c.q0 = q0;
        c.q1 = std::min(nq, q0 + chunk);
        for (int j = 0; j < 3; ++j) c.row0[j] = next[j];
        for (uint32_t q = c.q0; q < c.q1; ++q) ++c.n[kinds[q]];
        for (int kd = 0; kd < 3; ++kd) {
            c.map[kd] = at;
            at += (size_t)3 * c.n[kd];
        }
        uint32_t fill[3] = {0, 0, 0};
        for (uint32_t q = c.q0; q < c.q1; ++q) {
            const int kd = kinds[q], f = HYB_KIND_SRC[kd][0], s = HYB_KIND_SRC[kd][1];
            uint32_t *m = maps->data() + c.map[kd];
            const uint32_t i = fill[kd]++;
            m[i] = q - c.q0;
            m[c.n[kd] + i] = next[f]++ - c.row0[f];
            m[2 * (size_t)c.n[kd] + i] = next[s]++ - c.row0[s];
        }
        for (int j = 0; j < 3; ++j) c.rows[j] = next[j] - c.row0[j];
        chunks->push_back(c);
    }
}

cdb_status mixed_fuse(const MixedChunk &c, const RrfList lists[3], const uint32_t *d_maps, const uint8_t *d_err_dense, float k,
                      uint32_t ld_out, uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s) {
    for (int kd = 0; kd < 3; ++kd) {
        if (!c.n[kd]) continue;
        const int f = HYB_KIND_SRC[kd][0];
        const uint32_t *m = d_maps + c.map[kd];
        RrfList a = lists[f], b = lists[HYB_KIND_SRC[kd][1]];
        a.rows = m + c.n[kd];
        b.rows = m + 2 * (size_t)c.n[kd];
        const RrfRows o{m, f == 0 ? d_err_dense : nullptr, d_err};
        if (cdb_status rc = fuse_launch(a, b, c.n[kd], k, ld_out, d_ids, d_scores, d_counts, s, o)) return rc;
    }
    return CDB_OK;
}

namespace {

enum Source { SRC_DENSE = 0, SRC_SPARSE = 1, SRC_TFIDF = 2 };

// The sources a call searches, in list order (a pair: first, second; a mixed batch: dense, sparse, TF-IDF, those with
// queries), each over its own batch of nq[i] queries, and the fusions of their lists.
struct Plan {
    int n = 0;
    Source src[3];
    uint32_t nq[3];
    uint32_t ld[3];       // columns of each intermediate list
    int device = -1;
};

uint32_t source_ld(Source s, uint32_t top_k) { return s == SRC_TFIDF ? std::min(3 * top_k, TF_RESULTS) : 3 * top_k; }

int source_device(const cdb_hybrid_sources *h, Source s) {
    return s == SRC_DENSE ? index_device(h->dense) : s == SRC_SPARSE ? sparse_index_device(h->sparse) : tfidf_index_device(h->tfidf);
}

// the refusals shared by both forms of sources after the source list: sparse rerank bound, one device, no graph metadata
cdb_status plan_sources(const cdb_hybrid_sources *h, uint32_t top_k, Plan *p) {
    const uint32_t k3 = 3 * top_k;
    bool sparse = false;
    for (int j = 0; j < p->n; ++j) sparse |= p->src[j] == SRC_SPARSE;
    if (sparse && h->sparse_params.rerank)
        CDB_REQUIRE(h->sparse_params.reranking_factor >= 1 && (uint64_t)k3 * h->sparse_params.reranking_factor <= 5120,
                   "3 * top_k * reranking_factor must be in 1..5120");
    // the handles' devices (immutable after create)
    for (int j = 0; j < p->n; ++j) {
        const int d = source_device(h, p->src[j]);
        CDB_REQUIRE(!j || d == p->device, "the handles live on different devices");
        p->device = d;
    }
    for (int j = 0; j < p->n; ++j)
        if (p->src[j] == SRC_DENSE && index_has_graph_metadata(h->dense)) {
            set_error("a dense handle with graph metadata searches through cdb_search_batch_filtered: fuse with cdb_rrf_fuse");
            return CDB_UNSUPPORTED;
        }
    return CDB_OK;
}

// every refusal that needs no device: the handles are read only after the request itself is well-formed
cdb_status make_plan(const cdb_hybrid_sources *h, uint32_t nq, uint32_t top_k, Plan *p) {
    CDB_REQUIRE(h, "null sources");
    CDB_REQUIRE(top_k <= HYB_MAX_TOP_K, "top_k must be <= 341 (each sub-search takes 3 * top_k <= 1024)");
    const int n_src = (h->dense != nullptr) + (h->sparse != nullptr) + (h->tfidf != nullptr);
    CDB_REQUIRE(n_src == 2, "a hybrid search takes exactly two sources");
    // the reference's dense sub-search always has Some(3 * top_k): top_k None has no hybrid form
    CDB_REQUIRE(!h->dense || !(h->dense_params.flags & CDB_SEARCH_ALL_CANDIDATES),
                "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k");
    if (h->dense) p->src[p->n++] = SRC_DENSE;
    if (h->sparse) p->src[p->n++] = SRC_SPARSE;
    if (h->tfidf) p->src[p->n++] = SRC_TFIDF;
    for (int j = 0; j < p->n; ++j) {
        p->nq[j] = nq;
        p->ld[j] = source_ld(p->src[j], top_k);
    }
    CDB_REQUIRE(!h->dense || h->dense_queries || !nq, "null dense queries");
    CDB_REQUIRE(!h->sparse || h->sparse_offsets || !nq, "null sparse query offsets");
    CDB_REQUIRE(!h->tfidf || h->tfidf_offsets || !nq, "null tf-idf query offsets");
    return plan_sources(h, top_k, p);
}

// a mixed batch's sources as cdb_hybrid_sources, and its plan: the sources with queries, in the order dense, sparse, TF-IDF.
// host: the query CSRs are host arrays, checked too.  Every refusal of the request comes before a handle is read.
cdb_status make_mixed_plan(const cdb_hybrid_mixed_sources *m, uint32_t nq, uint32_t top_k, bool host, cdb_hybrid_sources *h, Plan *p) {
    CDB_REQUIRE(m, "null sources");
    CDB_REQUIRE(top_k <= HYB_MAX_TOP_K, "top_k must be <= 341 (each sub-search takes 3 * top_k <= 1024)");
    const uint32_t n_src[3] = {m->n_dense, m->n_sparse, m->n_tfidf};
    if (cdb_status rc = check_kinds(m->kinds, nq, n_src)) return rc;
    CDB_REQUIRE(!m->n_dense || !(m->dense_params.flags & CDB_SEARCH_ALL_CANDIDATES),
                "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k");
    CDB_REQUIRE(!m->n_dense || m->dense, "null dense handle");
    CDB_REQUIRE(!m->n_sparse || m->sparse, "null sparse handle");
    CDB_REQUIRE(!m->n_tfidf || m->tfidf, "null tf-idf handle");
    CDB_REQUIRE(!m->n_dense || m->dense_queries, "null dense queries");
    CDB_REQUIRE(!m->n_sparse || m->sparse_offsets, "null sparse query offsets");
    CDB_REQUIRE(!m->n_tfidf || m->tfidf_offsets, "null tf-idf query offsets");
    if (m->n_sparse && m->sparse_params.rerank)
        CDB_REQUIRE(m->sparse_params.reranking_factor >= 1 && (uint64_t)3 * top_k * m->sparse_params.reranking_factor <= 5120,
                   "3 * top_k * reranking_factor must be in 1..5120");
    if (host && m->n_sparse) {
        if (cdb_status rc = check_csr(m->sparse_offsets, m->n_sparse, "sparse_offsets")) return rc;
        CDB_REQUIRE((m->sparse_dims && m->sparse_values) || !m->sparse_offsets[m->n_sparse], "null sparse query pairs");
    }
    if (host && m->n_tfidf) {
        if (cdb_status rc = check_csr(m->tfidf_offsets, m->n_tfidf, "tfidf_offsets")) return rc;
        CDB_REQUIRE(m->tfidf_hashes || !m->tfidf_offsets[m->n_tfidf], "null tf-idf query hashes");
    }
    *h = cdb_hybrid_sources{m->dense, m->dense_queries, m->dense_params, m->sparse, m->sparse_offsets, m->sparse_dims,
                            m->sparse_values, m->sparse_params, m->tfidf, m->tfidf_offsets, m->tfidf_hashes};
    for (int j = 0; j < 3; ++j)
        if (n_src[j]) {
            p->src[p->n] = (Source)j;
            p->nq[p->n] = n_src[j];
            p->ld[p->n++] = source_ld((Source)j, top_k);
        }
    return plan_sources(h, top_k, p);
}

cdb_status run_source(const cdb_hybrid_sources *h, Source src, uint32_t nq, uint32_t k3, uint32_t *ids, float *scores,
                      uint32_t *counts, uint8_t *d_err, cudaStream_t s) {
    switch (src) {
    case SRC_DENSE: {
        cdb_search_params p = h->dense_params;
        p.k = k3;
        return cdb_search_batch_device(h->dense, h->dense_queries, nq, &p, ids, scores, counts, d_err, s);
    }
    case SRC_SPARSE: {
        cdb_sparse_search_params p = h->sparse_params;
        p.k = k3;
        return cdb_sparse_search_batch_device(h->sparse, h->sparse_offsets, h->sparse_dims, h->sparse_values, nq, &p, ids, scores,
                                              counts, s);
    }
    default:
        return cdb_tfidf_search_batch_device(h->tfidf, h->tfidf_offsets, h->tfidf_hashes, nq, k3, ids, scores, counts, s);
    }
}

// The composed search on `s` after make_plan / make_mixed_plan and cudaSetDevice; top_k >= 1, at least one source with
// queries.  Every source runs once: the first on the caller's stream, the others on side streams forked from it and joined
// back, so they overlap.  A pair (kinds null) fuses its two lists row by row, the dense search writing d_err itself; a mixed
// batch (kinds [nq]) fuses each kind present with one launch through its row maps, which also scatters the dense error
// bytes.  The lists, the maps and the dense error bytes live in one stream-ordered block, freed behind the last fusion.
cdb_status hybrid_device(const cdb_hybrid_sources *h, const Plan &p, const uint8_t *kinds, uint32_t nq, uint32_t top_k, float k,
                         uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s) {
    const uint32_t k3 = 3 * top_k;
    std::vector<MixedChunk> chunks;
    std::vector<uint32_t> maps;
    if (kinds) mixed_chunks(kinds, nq, std::max<uint32_t>(nq, 1), &chunks, &maps);
    size_t bytes = maps.size() * 4;
    uint32_t n_dense = 0;
    for (int j = 0; j < p.n; ++j) {
        bytes += (size_t)p.nq[j] * ((size_t)p.ld[j] * 8 + 4);
        if (p.src[j] == SRC_DENSE) n_dense = p.nq[j];
    }
    const bool err_scratch = kinds && d_err && n_dense;
    if (err_scratch) bytes += n_dense;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    // per list: ids, scores, counts; then the maps and the dense error bytes
    uint32_t *ids[3], *counts[3];
    float *scores[3];
    uint8_t *at = buf;
    for (int j = 0; j < p.n; ++j) {
        ids[j] = reinterpret_cast<uint32_t *>(at);
        scores[j] = reinterpret_cast<float *>(ids[j] + (size_t)p.nq[j] * p.ld[j]);
        counts[j] = reinterpret_cast<uint32_t *>(scores[j] + (size_t)p.nq[j] * p.ld[j]);
        at = reinterpret_cast<uint8_t *>(counts[j] + p.nq[j]);
    }
    uint32_t *d_maps = reinterpret_cast<uint32_t *>(at);
    uint8_t *err_dense = err_scratch ? reinterpret_cast<uint8_t *>(d_maps + maps.size()) : nullptr;
    cudaStream_t side[2] = {nullptr, nullptr};
    cudaEvent_t fork = nullptr, join[2] = {nullptr, nullptr};
    cudaError_t e = cudaSuccess;
    if (!maps.empty()) e = cudaMemcpyAsync(d_maps, maps.data(), maps.size() * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && p.n > 1) e = cudaEventCreateWithFlags(&fork, cudaEventDisableTiming);
    if (e == cudaSuccess && p.n > 1) e = cudaEventRecord(fork, s);
    for (int j = 1; j < p.n && e == cudaSuccess; ++j) {
        e = cudaStreamCreateWithFlags(&side[j - 1], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&join[j - 1], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(side[j - 1], fork, 0);
    }
    cdb_status rc = CDB_OK;
    if (e != cudaSuccess) {
        set_error(std::string("hybrid search: ") + cudaGetErrorString(e));
        rc = CDB_CUDA_ERROR;
    }
    // the first list on the caller's stream, the others on the side streams: the searches overlap
    for (int j = 0; j < p.n && !rc; ++j) {
        uint8_t *err = p.src[j] != SRC_DENSE ? nullptr : kinds ? err_dense : d_err;
        rc = run_source(h, p.src[j], p.nq[j], k3, ids[j], scores[j], counts[j], err, j ? side[j - 1] : s);
    }
    // joined whatever happened, so that the scratch is freed behind everything that was enqueued
    for (int j = 0; j < 2; ++j) {
        if (!side[j]) continue;
        bool joined = false;
        if (join[j]) {
            e = cudaEventRecord(join[j], side[j]);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(s, join[j], 0);
            joined = e == cudaSuccess;
        }
        if (!joined) {
            cudaStreamSynchronize(side[j]);
            if (!rc) {
                set_error(std::string("hybrid search: ") + cudaGetErrorString(e));
                rc = CDB_CUDA_ERROR;
            }
        }
    }
    if (!rc && !kinds) {
        const RrfList a{ids[0], counts[0], p.ld[0], 1}, b{ids[1], counts[1], p.ld[1], 1};
        rc = fuse_launch(a, b, nq, k, 6 * top_k, d_ids, d_scores, d_counts, s);
    } else if (!rc) {
        RrfList lists[3] = {};
        for (int j = 0; j < p.n; ++j) lists[p.src[j]] = RrfList{ids[j], counts[j], p.ld[j], 1};
        rc = mixed_fuse(chunks[0], lists, d_maps, err_dense, k, 6 * top_k, d_ids, d_scores, d_counts, d_err, s);
    }
    cudaFreeAsync(buf, s);
    // released once their pending work completes
    if (fork) cudaEventDestroy(fork);
    for (int j = 0; j < 2; ++j) {
        if (join[j]) cudaEventDestroy(join[j]);
        if (side[j]) cudaStreamDestroy(side[j]);
    }
    return rc;
}

}  // namespace
}  // namespace cdb

using namespace cdb;

extern "C" {

cdb_status cdb_rrf_fuse_device(int32_t device, const uint32_t *d_first_ids, const uint32_t *d_first_counts, uint32_t ld_first,
                               uint32_t first_id_stride, const uint32_t *d_second_ids, const uint32_t *d_second_counts,
                               uint32_t ld_second, uint32_t second_id_stride, uint32_t nq, float fusion_constant_k,
                               uint32_t ld_out, uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts, void *stream) {
    cdb_status rc = check_fuse_args(ld_first, ld_second, nq, ld_out, d_first_ids, d_first_counts, d_second_ids, d_second_counts,
                                    d_out_ids, d_out_scores, d_out_counts);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaSetDevice(device));
    const RrfList a{d_first_ids, d_first_counts, ld_first, first_id_stride}, b{d_second_ids, d_second_counts, ld_second, second_id_stride};
    return fuse_launch(a, b, nq, fusion_constant_k, ld_out, d_out_ids, d_out_scores, d_out_counts, (cudaStream_t)stream);
}

cdb_status cdb_rrf_fuse(int32_t device, const uint32_t *first_ids, const uint32_t *first_counts, uint32_t ld_first,
                        uint32_t first_id_stride, const uint32_t *second_ids, const uint32_t *second_counts, uint32_t ld_second,
                        uint32_t second_id_stride, uint32_t nq, float fusion_constant_k, uint32_t ld_out, uint32_t *out_ids,
                        float *out_scores, uint32_t *out_counts) {
    cdb_status rc = check_fuse_args(ld_first, ld_second, nq, ld_out, first_ids, first_counts, second_ids, second_counts, out_ids,
                                    out_scores, out_counts);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaSetDevice(device));
    if (!nq) return CDB_OK;
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    const size_t na = (size_t)nq * ld_first, nb = (size_t)nq * ld_second, no = (size_t)nq * ld_out;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, (na + nb + 2 * (size_t)nq + 2 * no + nq) * 4, s));
    uint32_t *d_a = reinterpret_cast<uint32_t *>(buf), *d_b = d_a + na, *d_ca = d_b + nb, *d_cb = d_ca + nq, *d_ids = d_cb + nq;
    float *d_scores = reinterpret_cast<float *>(d_ids + no);
    uint32_t *d_counts = reinterpret_cast<uint32_t *>(d_scores + no);
    cudaError_t e = cudaSuccess;
    if (na) e = cudaMemcpyAsync(d_a, first_ids, na * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nb) e = cudaMemcpyAsync(d_b, second_ids, nb * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_ca, first_counts, (size_t)nq * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_cb, second_counts, (size_t)nq * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) { set_error(std::string("rrf fuse: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) {
        const RrfList a{d_a, d_ca, ld_first, first_id_stride}, b{d_b, d_cb, ld_second, second_id_stride};
        rc = fuse_launch(a, b, nq, fusion_constant_k, ld_out, d_ids, d_scores, d_counts, s);
    }
    if (!rc) {
        if (no) e = cudaMemcpyAsync(out_ids, d_ids, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && no) e = cudaMemcpyAsync(out_scores, d_scores, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_counts, d_counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error(std::string("rrf fuse: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(buf, s);
    return rc;
}

cdb_status cdb_hybrid_search_batch_device(const cdb_hybrid_sources *sources, uint32_t nq, uint32_t top_k, float fusion_constant_k,
                                          uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err_flags, void *stream) {
    CDB_REQUIRE(!nq || !top_k || (d_ids && d_scores && d_counts), "null output");
    Plan p;
    cdb_status rc = make_plan(sources, nq, top_k, &p);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaSetDevice(p.device));
    if (!nq) return CDB_OK;
    cudaStream_t s = stream ? (cudaStream_t)stream : cudaStreamLegacy;
    if (!top_k) {
        CDB_CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, s));
        return CDB_OK;
    }
    return hybrid_device(sources, p, nullptr, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, d_err_flags, s);
}

cdb_status cdb_hybrid_search_batch(const cdb_hybrid_sources *sources, uint32_t nq, uint32_t top_k, float fusion_constant_k,
                                   uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(!nq || (out_counts && (!top_k || (out_ids && out_scores))), "null output");
    Plan p;
    cdb_status rc = make_plan(sources, nq, top_k, &p);
    if (rc) return rc;
    const cdb_hybrid_sources &h = *sources;
    uint64_t sp_pairs = 0, tf_hashes = 0;
    if (nq && h.sparse) {
        if ((rc = check_csr(h.sparse_offsets, nq, "sparse_offsets"))) return rc;
        sp_pairs = h.sparse_offsets[nq];
        CDB_REQUIRE((h.sparse_dims && h.sparse_values) || !sp_pairs, "null sparse query pairs");
    }
    if (nq && h.tfidf) {
        if ((rc = check_csr(h.tfidf_offsets, nq, "tfidf_offsets"))) return rc;
        tf_hashes = h.tfidf_offsets[nq];
        CDB_REQUIRE(h.tfidf_hashes || !tf_hashes, "null tf-idf query hashes");
    }
    CDB_CUDA_TRY(cudaSetDevice(p.device));
    if (!nq) return CDB_OK;
    if (!top_k) {
        memset(out_counts, 0, (size_t)nq * 4);
        return CDB_OK;
    }
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    // one buffer: dense queries, sparse CSR, tf-idf CSR, then the outputs (8-byte parts first)
    const size_t dq = h.dense ? (size_t)nq * index_dim(h.dense) : 0;
    const size_t ld_out = 6 * (size_t)top_k, no = (size_t)nq * ld_out;
    const size_t n_sp_off = h.sparse ? nq + 1 : 0, n_tf_off = h.tfidf ? nq + 1 : 0;
    const size_t bytes = (n_sp_off + n_tf_off) * 8 + (dq + 2 * sp_pairs + tf_hashes + 2 * no + nq) * 4 + nq;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    cdb_hybrid_sources d = h;
    uint64_t *sp_off = reinterpret_cast<uint64_t *>(buf), *tf_off = sp_off + n_sp_off;
    float *dense_q = reinterpret_cast<float *>(tf_off + n_tf_off);
    uint32_t *sp_dims = reinterpret_cast<uint32_t *>(dense_q + dq);
    float *sp_vals = reinterpret_cast<float *>(sp_dims + sp_pairs);
    uint32_t *tf_h = reinterpret_cast<uint32_t *>(sp_vals + sp_pairs);
    uint32_t *d_ids = tf_h + tf_hashes;
    float *d_scores = reinterpret_cast<float *>(d_ids + no);
    uint32_t *d_counts = reinterpret_cast<uint32_t *>(d_scores + no);
    uint8_t *d_err = reinterpret_cast<uint8_t *>(d_counts + nq);
    cudaError_t e = cudaSuccess;
    if (h.dense) {
        e = cudaMemcpyAsync(dense_q, h.dense_queries, dq * 4, cudaMemcpyHostToDevice, s);
        d.dense_queries = dense_q;
    }
    if (h.sparse) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(sp_off, h.sparse_offsets, n_sp_off * 8, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && sp_pairs) e = cudaMemcpyAsync(sp_dims, h.sparse_dims, sp_pairs * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && sp_pairs) e = cudaMemcpyAsync(sp_vals, h.sparse_values, sp_pairs * 4, cudaMemcpyHostToDevice, s);
        d.sparse_offsets = sp_off;
        d.sparse_dims = sp_dims;
        d.sparse_values = sp_vals;
    }
    if (h.tfidf) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(tf_off, h.tfidf_offsets, n_tf_off * 8, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && tf_hashes) e = cudaMemcpyAsync(tf_h, h.tfidf_hashes, tf_hashes * 4, cudaMemcpyHostToDevice, s);
        d.tfidf_offsets = tf_off;
        d.tfidf_hashes = tf_h;
    }
    if (e != cudaSuccess) { set_error(std::string("hybrid search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) rc = hybrid_device(&d, p, nullptr, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, d_err, s);
    if (!rc) {
        e = cudaMemcpyAsync(out_ids, d_ids, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_scores, d_scores, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_counts, d_counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && err_flags && h.dense) e = cudaMemcpyAsync(err_flags, d_err, nq, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error(std::string("hybrid search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(buf, s);
    return rc;
}

cdb_status cdb_hybrid_search_batch_mixed_device(const cdb_hybrid_mixed_sources *sources, uint32_t nq, uint32_t top_k,
                                                float fusion_constant_k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                                uint8_t *d_err_flags, void *stream) {
    CDB_REQUIRE(!nq || (d_counts && (!top_k || (d_ids && d_scores))), "null output");
    Plan p;
    cdb_hybrid_sources h;
    cdb_status rc = make_mixed_plan(sources, nq, top_k, false, &h, &p);
    if (rc || !nq) return rc;
    CDB_CUDA_TRY(cudaSetDevice(p.device));
    cudaStream_t s = stream ? (cudaStream_t)stream : cudaStreamLegacy;
    if (!top_k) {
        CDB_CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, s));
        return CDB_OK;
    }
    return hybrid_device(&h, p, sources->kinds, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, d_err_flags, s);
}

cdb_status cdb_hybrid_search_batch_mixed(const cdb_hybrid_mixed_sources *sources, uint32_t nq, uint32_t top_k, float fusion_constant_k,
                                         uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(!nq || (out_counts && (!top_k || (out_ids && out_scores))), "null output");
    Plan p;
    cdb_hybrid_sources h;
    cdb_status rc = make_mixed_plan(sources, nq, top_k, true, &h, &p);
    if (rc) return rc;
    const cdb_hybrid_mixed_sources &m = *sources;
    const uint64_t sp_pairs = m.n_sparse ? m.sparse_offsets[m.n_sparse] : 0, tf_hashes = m.n_tfidf ? m.tfidf_offsets[m.n_tfidf] : 0;
    if (!nq) return CDB_OK;
    if (!top_k) {
        memset(out_counts, 0, (size_t)nq * 4);
        return CDB_OK;
    }
    CDB_CUDA_TRY(cudaSetDevice(p.device));
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    // one buffer: dense queries, sparse CSR, tf-idf CSR, then the outputs (8-byte parts first)
    const size_t dq = m.n_dense ? (size_t)m.n_dense * index_dim(m.dense) : 0;
    const size_t ld_out = 6 * (size_t)top_k, no = (size_t)nq * ld_out;
    const size_t n_sp_off = m.n_sparse ? m.n_sparse + 1 : 0, n_tf_off = m.n_tfidf ? m.n_tfidf + 1 : 0;
    const size_t bytes = (n_sp_off + n_tf_off) * 8 + (dq + 2 * sp_pairs + tf_hashes + 2 * no + nq) * 4 + nq;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    uint64_t *sp_off = reinterpret_cast<uint64_t *>(buf), *tf_off = sp_off + n_sp_off;
    float *dense_q = reinterpret_cast<float *>(tf_off + n_tf_off);
    uint32_t *sp_dims = reinterpret_cast<uint32_t *>(dense_q + dq);
    float *sp_vals = reinterpret_cast<float *>(sp_dims + sp_pairs);
    uint32_t *tf_h = reinterpret_cast<uint32_t *>(sp_vals + sp_pairs);
    uint32_t *d_ids = tf_h + tf_hashes;
    float *d_scores = reinterpret_cast<float *>(d_ids + no);
    uint32_t *d_counts = reinterpret_cast<uint32_t *>(d_scores + no);
    uint8_t *d_err = reinterpret_cast<uint8_t *>(d_counts + nq);
    cudaError_t e = cudaSuccess;
    if (dq) e = cudaMemcpyAsync(dense_q, m.dense_queries, dq * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_sp_off) e = cudaMemcpyAsync(sp_off, m.sparse_offsets, n_sp_off * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && sp_pairs) e = cudaMemcpyAsync(sp_dims, m.sparse_dims, sp_pairs * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && sp_pairs) e = cudaMemcpyAsync(sp_vals, m.sparse_values, sp_pairs * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_tf_off) e = cudaMemcpyAsync(tf_off, m.tfidf_offsets, n_tf_off * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && tf_hashes) e = cudaMemcpyAsync(tf_h, m.tfidf_hashes, tf_hashes * 4, cudaMemcpyHostToDevice, s);
    h.dense_queries = dense_q;
    h.sparse_offsets = sp_off;
    h.sparse_dims = sp_dims;
    h.sparse_values = sp_vals;
    h.tfidf_offsets = tf_off;
    h.tfidf_hashes = tf_h;
    if (e != cudaSuccess) { set_error(std::string("hybrid search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) rc = hybrid_device(&h, p, m.kinds, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, err_flags ? d_err : nullptr, s);
    if (!rc) {
        e = cudaMemcpyAsync(out_ids, d_ids, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_scores, d_scores, no * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_counts, d_counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && err_flags) e = cudaMemcpyAsync(err_flags, d_err, nq, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error(std::string("hybrid search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(buf, s);
    return rc;
}

}  // extern "C"
