// hybrid.cu -- hybrid search (hybrid_search / batch_hybrid_search, src/api/vectordb/search/repo.rs:168-555): reciprocal-rank
// fusion of two ranked lists per query, and the composed search that runs two of the dense, sparse and TF-IDF searches and
// fuses their results on the device.  The contract is the header comment of cdb_rrf_fuse (DESIGN.md section 8e).
// check_fuse_args and fuse_launch also serve a shard group's hybrid search (shard_group.cu, DESIGN.md section 8h).
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

__global__ void __launch_bounds__(1024) rrf_fuse_kernel(RrfList a, RrfList b, float k, uint32_t n_sort, uint32_t ld_out,
                                                        uint32_t *__restrict__ out_ids, float *__restrict__ out_scores,
                                                        uint32_t *__restrict__ out_counts) {
    __shared__ uint64_t ent[RRF_MAX];   // (key << 32 | list << 31 | rank), ascending; ~0 = no entry
    __shared__ uint64_t res[RRF_MAX];   // (order_key(score) << 32 | ~key), descending; 0 = no key
    __shared__ uint32_t s_cnt;
    const uint32_t q = blockIdx.x, tid = threadIdx.x;
    const uint32_t na = min(a.counts[q], a.ld), nb = min(b.counts[q], b.ld), n = na + nb;
    if (tid == 0) s_cnt = 0;
    for (uint32_t i = tid; i < n_sort; i += blockDim.x) {
        uint64_t e = ~0ull;
        if (i < na)
            e = ((uint64_t)rrf_key(a.ids[(size_t)q * a.ld + i], a.stride) << 32) | i;
        else if (i >= a.ld && i - a.ld < nb)
            e = ((uint64_t)rrf_key(b.ids[(size_t)q * b.ld + (i - a.ld)], b.stride) << 32) | (1u << 31) | (i - a.ld);
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
                       uint32_t *d_counts, cudaStream_t s) {
    if (!nq) return CDB_OK;
    uint32_t n_sort = 2;
    while (n_sort < a.ld + b.ld) n_sort <<= 1;
    const uint32_t threads = std::min<uint32_t>(1024, std::max<uint32_t>(32, n_sort / 2));
    rrf_fuse_kernel<<<nq, threads, 0, s>>>(a, b, k, n_sort, ld_out, d_ids, d_scores, d_counts);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

namespace {

enum Source { SRC_DENSE = 0, SRC_SPARSE = 1, SRC_TFIDF = 2 };

struct Plan {
    Source src[2];        // first list, second list
    uint32_t ld[2];       // columns of each intermediate list
    int device;
};

// every refusal that needs no device: the handles are read only after the request itself is well-formed
cdb_status make_plan(const cdb_hybrid_sources *h, uint32_t nq, uint32_t top_k, Plan *p) {
    CDB_REQUIRE(h, "null sources");
    CDB_REQUIRE(top_k <= HYB_MAX_TOP_K, "top_k must be <= 341 (each sub-search takes 3 * top_k <= 1024)");
    const int n_src = (h->dense != nullptr) + (h->sparse != nullptr) + (h->tfidf != nullptr);
    CDB_REQUIRE(n_src == 2, "a hybrid search takes exactly two sources");
    // the reference's dense sub-search always has Some(3 * top_k): top_k None has no hybrid form
    CDB_REQUIRE(!h->dense || !(h->dense_params.flags & CDB_SEARCH_ALL_CANDIDATES),
                "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k");
    const uint32_t k3 = 3 * top_k;
    int i = 0;
    if (h->dense) { p->src[i] = SRC_DENSE; p->ld[i++] = k3; }
    if (h->sparse) { p->src[i] = SRC_SPARSE; p->ld[i++] = k3; }
    if (h->tfidf) { p->src[i] = SRC_TFIDF; p->ld[i++] = std::min(k3, TF_RESULTS); }
    CDB_REQUIRE(!h->dense || h->dense_queries || !nq, "null dense queries");
    CDB_REQUIRE(!h->sparse || h->sparse_offsets || !nq, "null sparse query offsets");
    CDB_REQUIRE(!h->tfidf || h->tfidf_offsets || !nq, "null tf-idf query offsets");
    if (h->sparse && h->sparse_params.rerank)
        CDB_REQUIRE(h->sparse_params.reranking_factor >= 1 && (uint64_t)k3 * h->sparse_params.reranking_factor <= 5120,
                   "3 * top_k * reranking_factor must be in 1..5120");
    // the handles' devices (immutable after create)
    int dev[2];
    for (int j = 0; j < 2; ++j)
        dev[j] = p->src[j] == SRC_DENSE ? index_device(h->dense)
               : p->src[j] == SRC_SPARSE ? sparse_index_device(h->sparse) : tfidf_index_device(h->tfidf);
    CDB_REQUIRE(dev[0] == dev[1], "the two handles live on different devices");
    p->device = dev[0];
    if (h->dense && index_has_graph_metadata(h->dense)) {
        set_error("a dense handle with graph metadata searches through cdb_search_batch_filtered: fuse with cdb_rrf_fuse");
        return CDB_UNSUPPORTED;
    }
    return CDB_OK;
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

// the composed search on `s` after make_plan and cudaSetDevice; top_k >= 1, nq >= 1
cdb_status hybrid_device(const cdb_hybrid_sources *h, const Plan &p, uint32_t nq, uint32_t top_k, float k, uint32_t *d_ids,
                         float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s) {
    const uint32_t k3 = 3 * top_k;
    const size_t cols = (size_t)p.ld[0] + p.ld[1];
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, (size_t)nq * (cols * 8 + 8), s));
    uint32_t *ids[2], *counts[2];
    float *scores[2];
    ids[0] = reinterpret_cast<uint32_t *>(buf);
    ids[1] = ids[0] + (size_t)nq * p.ld[0];
    scores[0] = reinterpret_cast<float *>(ids[1] + (size_t)nq * p.ld[1]);
    scores[1] = scores[0] + (size_t)nq * p.ld[0];
    counts[0] = reinterpret_cast<uint32_t *>(scores[1] + (size_t)nq * p.ld[1]);
    counts[1] = counts[0] + nq;
    cudaStream_t side = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&fork, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&join, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(fork, s);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(side, fork, 0);
    cdb_status rc = CDB_OK;
    if (e != cudaSuccess) {
        set_error(std::string("hybrid search: ") + cudaGetErrorString(e));
        rc = CDB_CUDA_ERROR;
    }
    // the first list on the caller's stream, the second on the side stream: the two searches overlap
    if (!rc) rc = run_source(h, p.src[0], nq, k3, ids[0], scores[0], counts[0], p.src[0] == SRC_DENSE ? d_err : nullptr, s);
    if (!rc) rc = run_source(h, p.src[1], nq, k3, ids[1], scores[1], counts[1], nullptr, side);
    // joined whatever happened, so that the scratch is freed behind everything that was enqueued
    bool joined = false;
    if (side && join) {
        e = cudaEventRecord(join, side);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(s, join, 0);
        joined = e == cudaSuccess;
    }
    if (side && !joined) cudaStreamSynchronize(side);
    if (!joined && !rc) {
        set_error(std::string("hybrid search: ") + cudaGetErrorString(e));
        rc = CDB_CUDA_ERROR;
    }
    if (!rc) {
        const RrfList a{ids[0], counts[0], p.ld[0], 1}, b{ids[1], counts[1], p.ld[1], 1};
        rc = fuse_launch(a, b, nq, k, 6 * top_k, d_ids, d_scores, d_counts, s);
    }
    cudaFreeAsync(buf, s);
    // released once their pending work completes
    if (fork) cudaEventDestroy(fork);
    if (join) cudaEventDestroy(join);
    if (side) cudaStreamDestroy(side);
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
    return hybrid_device(sources, p, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, d_err_flags, s);
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
    if (!rc) rc = hybrid_device(&d, p, nq, top_k, fusion_constant_k, d_ids, d_scores, d_counts, d_err, s);
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

}  // extern "C"
