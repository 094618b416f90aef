// shard_group.cu -- row-sharded search over the GPUs of one node behind the C ABI (SURVEY 8e; the reference's call site is
// IndexOps::batch_search, src/indexes/mod.rs:260-272 -- one process, rayon over queries; here one index shard per GPU).
//
// Every shard searches the same query batch; its final kernel (exact re-rank / merge / key selection) writes the packed
// 64-bit selection keys (order_key(score) << 32 | ~global_id, best first, 0 = empty) of every query STRAIGHT INTO ITS SLOT of
// the gather buffer, the per-query error bytes right behind them; ONE ncclAllGather of B*k*8 (+ B) bytes per rank makes
// every rank hold all slots; one merge kernel picks the global top-k per query with the common ordering rule.  No
// id/score arrays are exchanged, no pack kernel, no second collective.
//
// Two deployments, same code:
//   cdb_shard_group_create       one process, n devices (ncclCommInitAll); the host calls cdb_search_batch_sharded once
//   cdb_shard_group_create_rank  one process per GPU (torchrun style; rank 0 distributes cdb_nccl_unique_id())
// NCCL is bound at run time (dlopen of libnccl.so.2, the copy already in the process if there is one), so the library
// itself has no NCCL link dependency and a single-GPU host never needs it.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <string>
#include <vector>

#include "kernels.h"

struct cdb_index;
namespace cdb {
cdb_status index_search_device_keys(cdb_index *ix, const float *d_queries, uint32_t nq, const cdb_search_params *p, uint32_t *d_ids,
                                    float *d_scores, uint32_t *d_counts, uint8_t *d_err, uint64_t *d_keys, cudaStream_t s,
                                    const ShardFilters *f);
cdb_status index_check_all_width(cdb_index *ix, uint32_t w);
uint32_t index_md_dims(cdb_index *ix);
int index_device(const cdb_index *ix);
uint32_t index_dim(const cdb_index *ix);
int index_metric(const cdb_index *ix);
int index_storage_type(const cdb_index *ix);
uint32_t index_id_base(const cdb_index *ix);
uint64_t index_capacity(const cdb_index *ix);
int index_result_metric(const cdb_index *ix, int mode);

// sparse.cu: a shard group's two-phase sparse search
std::shared_mutex &sparse_index_mutex(cdb_sparse_index *ix);
int sparse_index_device(const cdb_sparse_index *ix);
uint32_t sparse_index_bits(const cdb_sparse_index *ix);
float sparse_index_upper_bound(const cdb_sparse_index *ix);
uint32_t sparse_index_id_base(const cdb_sparse_index *ix);
uint64_t sparse_index_capacity(const cdb_sparse_index *ix);
cdb_status sparse_check_params(const cdb_sparse_search_params *p, uint32_t *m);
cdb_status sparse_shard_select(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                               const cdb_sparse_search_params *p, uint32_t m, uint64_t *keys, uint32_t *cnt, cudaStream_t s);
cdb_status sparse_group_select(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t m, uint64_t *keys,
                               uint32_t *cnt, cudaStream_t s);
cdb_status sparse_shard_rerank(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                               uint32_t m, const uint64_t *keys, const uint32_t *cnt, uint64_t *out, cudaStream_t s);
cdb_status sparse_group_finalize(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t m, uint32_t k, int rerank,
                                 uint64_t *keys, const uint32_t *cnt, uint32_t *ids, float *scores, uint32_t *counts, cudaStream_t s);
cdb_status sparse_group_merge_all(const uint64_t *gathered, size_t words, uint32_t world, const uint32_t *d_pre, uint32_t nb, uint32_t n,
                                  int rerank, uint32_t *ids, float *scores, cudaStream_t s);

// tfidf.cu: a shard group's TF-IDF search under the group's idf
std::shared_mutex &tfidf_index_mutex(cdb_tfidf_index *ix);
int tfidf_index_device(const cdb_tfidf_index *ix);
uint32_t tfidf_index_id_base(const cdb_tfidf_index *ix);
uint64_t tfidf_index_capacity(const cdb_tfidf_index *ix);
uint32_t tfidf_out_cols(uint32_t k);
cdb_status tfidf_shard_stats(const cdb_tfidf_index *ix, const uint32_t *d_qhash, uint64_t n_qh, uint32_t *out, cudaStream_t s);
cdb_status tfidf_group_idf(const uint64_t *gathered, size_t words, uint32_t world, uint64_t n_qh, float *q_idf, cudaStream_t s);
cdb_status tfidf_shard_winners(cdb_tfidf_index *ix, const uint64_t *d_qoff, const uint32_t *d_qhash, uint64_t n_qh, const float *d_qidf, uint32_t nq,
                               uint2 *out, cudaStream_t s);
cdb_status tfidf_group_finalize(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t k, uint32_t *ids, float *scores,
                                uint32_t *counts, cudaStream_t s);

namespace {
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi *nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy a host framework already loaded, if any
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        api.h = h;
#define CDB_NCCL_SYM(field, name) api.field = reinterpret_cast<decltype(api.field)>(dlsym(h, name))
        CDB_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
        CDB_NCCL_SYM(CommInitRank, "ncclCommInitRank");
        CDB_NCCL_SYM(CommInitAll, "ncclCommInitAll");
        CDB_NCCL_SYM(CommDestroy, "ncclCommDestroy");
        CDB_NCCL_SYM(AllGather, "ncclAllGather");
        CDB_NCCL_SYM(GroupStart, "ncclGroupStart");
        CDB_NCCL_SYM(GroupEnd, "ncclGroupEnd");
        CDB_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef CDB_NCCL_SYM
        if (!api.GetUniqueId || !api.CommInitRank || !api.CommInitAll || !api.CommDestroy || !api.AllGather || !api.GroupStart ||
            !api.GroupEnd || !api.GetErrorString)
            api.h = nullptr;
    });
    return api.h ? &api : nullptr;
}
#define CDB_NCCL_TRY(api, expr)                                                                       \
    do {                                                                                              \
        ncclResult_t _r = (expr);                                                                     \
        if (_r != ncclSuccess) {                                                                      \
            set_error(std::string(#expr) + ": " + (api)->GetErrorString(_r));                         \
            return CDB_NCCL_ERROR;                                                                    \
        }                                                                                             \
    } while (0)

struct Buf {
    void *p = nullptr;
    size_t cap = 0;
    cdb_status ensure(size_t bytes) {
        if (bytes <= cap) return CDB_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        CDB_CUDA_TRY(cudaMalloc(&p, bytes + bytes / 4 + 256));
        cap = bytes + bytes / 4 + 256;
        return CDB_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// per-rank slot of the gather buffer, in u64 words: nq*k keys, then the nq error bytes
__host__ __device__ inline size_t slot_words(uint32_t nq, uint32_t k) { return (size_t)nq * k + ((size_t)nq + 7) / 8; }

// one CTA per query: the best k of world*k keys (rank selection; keys are unique), error bytes OR-ed over the ranks
__global__ void merge_gathered_kernel(const uint64_t *__restrict__ gathered, uint32_t world, uint32_t nq, uint32_t k, size_t words,
                                      int metric, uint32_t *__restrict__ ids, float *__restrict__ scores,
                                      uint32_t *__restrict__ counts, uint8_t *__restrict__ err) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    __shared__ int nvalid;
    const uint32_t q = blockIdx.x, M = world * k;
    if (threadIdx.x == 0) nvalid = 0;
    for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) { ids[(size_t)q * k + j] = CDB_INVALID_ID; scores[(size_t)q * k + j] = 0.0f; }
    __syncthreads();
    int local = 0;
    for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) {
        const uint32_t r = i / k, j = i - r * k;
        const uint64_t v = gathered[(size_t)r * words + (size_t)q * k + j];
        keys[i] = v;
        local += v != 0;
    }
    if (local) atomicAdd(&nvalid, local);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) {
        const uint64_t key = keys[i];
        if (!key) continue;
        uint32_t rank = 0;
        for (uint32_t j = 0; j < M; ++j) rank += keys[j] > key;
        if (rank < k) {
            ids[(size_t)q * k + rank] = key64_id(key);
            scores[(size_t)q * k + rank] = __uint_as_float(key_to_bits(metric, (uint32_t)(key >> 32)));
        }
    }
    if (threadIdx.x == 0) {
        if (counts) counts[q] = (uint32_t)nvalid < k ? (uint32_t)nvalid : k;
        if (err) {
            uint8_t e = 0;
            for (uint32_t r = 0; r < world; ++r) e |= reinterpret_cast<const uint8_t *>(gathered + (size_t)r * words + (size_t)nq * k)[q];
            err[q] = e;
        }
    }
}

// top_k None: one CTA per query merges `world` runs of w keys (each sorted descending, zero padded) into one sorted row of
// W = world * w columns.  An entry's position is its index in its run plus, for every other run, the number of that run's
// keys greater than it (binary search over all w slots: a zero key is never greater), so neither the run length nor the
// world size has a shared-memory bound.  The row is filled with CDB_INVALID_ID / 0 first: keys are unique (the shards' id
// ranges, and their replica ids, are disjoint), so the counts[q] = the number of non-zero keys land on [0, counts[q]), and a
// violated precondition leaves empty slots rather than stale ones.  Error bytes OR-ed over the ranks.
__global__ void merge_runs_kernel(const uint64_t *__restrict__ gathered, uint32_t world, uint32_t nq, uint32_t w, size_t words,
                                  int metric, uint32_t *__restrict__ ids, float *__restrict__ scores, uint32_t *__restrict__ counts,
                                  uint8_t *__restrict__ err) {
    __shared__ uint32_t total;
    const uint32_t q = blockIdx.x, W = world * w;
    auto run = [&](uint32_t r) { return gathered + (size_t)r * words + (size_t)q * w; };
    if (threadIdx.x == 0) total = 0;
    for (uint32_t o = threadIdx.x; o < W; o += blockDim.x) { ids[(size_t)q * W + o] = CDB_INVALID_ID; scores[(size_t)q * W + o] = 0.0f; }
    __syncthreads();
    uint32_t mine = 0;
    for (uint32_t i = threadIdx.x; i < W; i += blockDim.x) {
        const uint32_t r = i / w, j = i - r * w;
        const uint64_t key = run(r)[j];
        if (!key) continue;
        ++mine;
        uint32_t pos = j;
        for (uint32_t o = 0; o < world; ++o) {
            if (o == r) continue;
            const uint64_t *R = run(o);
            uint32_t lo = 0, hi = w;   // keys of run o greater than `key`
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (R[mid] > key) lo = mid + 1; else hi = mid;
            }
            pos += lo;
        }
        ids[(size_t)q * W + pos] = key64_id(key);
        scores[(size_t)q * W + pos] = __uint_as_float(key_to_bits(metric, (uint32_t)(key >> 32)));
    }
    if (mine) atomicAdd(&total, mine);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint8_t e = 0;
        for (uint32_t r = 0; r < world; ++r) e |= reinterpret_cast<const uint8_t *>(gathered + (size_t)r * words + (size_t)nq * w)[q];
        if (counts) counts[q] = total;
        if (err) err[q] = e;
    }
}
}  // namespace
}  // namespace cdb

using namespace cdb;

struct cdb_shard_group {
    uint32_t world = 1, rank0 = 0;        // ranks in the communicator; global rank of local slot 0
    bool loopback = false;                // local group with a repeated device: gather by device copies (tests on one GPU)
    std::vector<int> dev;                 // per local slot
    std::vector<ncclComm_t> comm;
    std::vector<cdb_index *> shard;
    std::vector<cdb_sparse_index *> sparse;   // a slot may hold a dense, a sparse and a TF-IDF shard at once
    std::vector<cdb_tfidf_index *> tfidf;
    std::vector<cudaStream_t> stream;
    std::vector<cudaEvent_t> ev;
    std::vector<Buf> gather, q, ids, scores, counts, rows, sel;   // rows: a host form's final rows (slot 0)
    std::mutex mu;
};

static cdb_status group_alloc_slots(cdb_shard_group *g, size_t n) {
    g->comm.assign(n, nullptr);
    g->shard.assign(n, nullptr);
    g->sparse.assign(n, nullptr);
    g->tfidf.assign(n, nullptr);
    g->stream.assign(n, nullptr);
    g->ev.assign(n, nullptr);
    g->gather.resize(n); g->q.resize(n); g->ids.resize(n); g->scores.resize(n); g->counts.resize(n); g->rows.resize(n); g->sel.resize(n);
    for (size_t i = 0; i < n; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        CDB_CUDA_TRY(cudaStreamCreateWithFlags(&g->stream[i], cudaStreamNonBlocking));
        CDB_CUDA_TRY(cudaEventCreateWithFlags(&g->ev[i], cudaEventDisableTiming));
    }
    return CDB_OK;
}

// ---------------------------------------------------------------- the host forms' staging: queries in, final rows out

struct HostArray {
    const void *h;
    size_t bytes;   // 0: not copied
};

// where a host form's query arrays landed: array j on local slot i at base[i] + off[j]
struct Staged {
    std::vector<uint8_t *> base;
    std::vector<size_t> off;
    template <class T> const T *at(size_t i, size_t j) const { return reinterpret_cast<const T *>(base[i] + off[j]); }
};

// The host arrays a into every local slot's q buffer, each 16-byte aligned behind the one before, on the slot's stream.
// Loopback: slot 0's stream then joins every slot's, since it may read any slot's queries (the sparse re-rank).
static cdb_status stage_queries(cdb_shard_group *g, const std::vector<HostArray> &a, Staged *st) {
    size_t bytes = 0;
    for (const HostArray &x : a) {
        st->off.push_back(bytes);
        bytes += (x.bytes + 15) & ~(size_t)15;
    }
    cdb_status rc;
    for (size_t i = 0; i < g->dev.size(); ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = g->q[i].ensure(bytes))) return rc;
        st->base.push_back(reinterpret_cast<uint8_t *>(g->q[i].p));
        for (size_t j = 0; j < a.size(); ++j)
            if (a[j].bytes)
                CDB_CUDA_TRY(cudaMemcpyAsync(st->base[i] + st->off[j], a[j].h, a[j].bytes, cudaMemcpyHostToDevice, g->stream[i]));
    }
    if (g->loopback) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        for (size_t i = 1; i < g->dev.size(); ++i) {
            CDB_CUDA_TRY(cudaEventRecord(g->ev[i], g->stream[i]));
            CDB_CUDA_TRY(cudaStreamWaitEvent(g->stream[0], g->ev[i], 0));
        }
    }
    return CDB_OK;
}

// A host form's final rows on slot 0, carved from g->rows[0] (the shards' own buffers hold their local results): ids and
// scores [nq][w], counts [nq], error bytes [nq]; and the caller's arrays they go to (null counts / err: not copied).
struct HostRows {
    size_t nq = 0, nk = 0;
    uint32_t *ids = nullptr, *counts = nullptr;
    float *scores = nullptr;
    uint8_t *err = nullptr;
    uint32_t *h_ids = nullptr, *h_counts = nullptr;
    float *h_scores = nullptr;
    uint8_t *h_err = nullptr;
};

static cdb_status host_rows(cdb_shard_group *g, uint32_t nq, uint32_t w, uint32_t *h_ids, float *h_scores, uint32_t *h_counts,
                            uint8_t *h_err, HostRows *r) {
    const size_t nk = (size_t)nq * w;
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    if (cdb_status rc = g->rows[0].ensure(nk * 8 + (size_t)nq * 8)) return rc;
    r->nq = nq;
    r->nk = nk;
    r->ids = reinterpret_cast<uint32_t *>(g->rows[0].p);
    r->scores = reinterpret_cast<float *>(r->ids + nk);
    r->counts = reinterpret_cast<uint32_t *>(r->scores + nk);
    r->err = reinterpret_cast<uint8_t *>(r->counts + nq);
    r->h_ids = h_ids; r->h_scores = h_scores; r->h_counts = h_counts; r->h_err = h_err;
    return CDB_OK;
}

static cdb_status copy_rows(cdb_shard_group *g, const HostRows &r) {
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    const cudaStream_t s0 = g->stream[0];
    CDB_CUDA_TRY(cudaMemcpyAsync(r.h_ids, r.ids, r.nk * 4, cudaMemcpyDeviceToHost, s0));
    CDB_CUDA_TRY(cudaMemcpyAsync(r.h_scores, r.scores, r.nk * 4, cudaMemcpyDeviceToHost, s0));
    if (r.h_counts) CDB_CUDA_TRY(cudaMemcpyAsync(r.h_counts, r.counts, r.nq * 4, cudaMemcpyDeviceToHost, s0));
    if (r.h_err) CDB_CUDA_TRY(cudaMemcpyAsync(r.h_err, r.err, r.nq, cudaMemcpyDeviceToHost, s0));
    return CDB_OK;
}

// The end of every host form, whatever rc says: the final rows r (if any) are copied back when the search was enqueued,
// then every local stream drains, collectives included, before the caller's locks and host buffers go.  The first error.
static cdb_status host_finish(cdb_shard_group *g, cdb_status rc, const HostRows *r) {
    if (!rc && r) rc = copy_rows(g, *r);
    for (size_t i = 0; i < g->dev.size(); ++i) {
        cudaSetDevice(g->dev[i]);
        const cudaError_t e = cudaStreamSynchronize(g->stream[i]);
        if (e != cudaSuccess && !rc) { set_error(std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    return rc;
}

extern "C" {

cdb_status cdb_nccl_unique_id(uint8_t *out_id128) {
    CDB_REQUIRE(out_id128, "null argument");
    NcclApi *n = nccl_api();
    if (!n) { set_error("libnccl.so.2 not found"); return CDB_NCCL_ERROR; }
    ncclUniqueId id;
    CDB_NCCL_TRY(n, n->GetUniqueId(&id));
    static_assert(sizeof(id) == CDB_NCCL_UNIQUE_ID_BYTES, "ncclUniqueId size");
    memcpy(out_id128, &id, sizeof(id));
    return CDB_OK;
}

cdb_status cdb_shard_group_create(const int32_t *device_ordinals, uint32_t n_devices, cdb_shard_group **out) {
    CDB_REQUIRE(device_ordinals && out && n_devices >= 1 && n_devices <= 64, "bad argument");
    std::unique_ptr<cdb_shard_group> g(new cdb_shard_group());
    g->world = n_devices;
    g->dev.assign(device_ordinals, device_ordinals + n_devices);
    for (uint32_t i = 0; i < n_devices; ++i)
        for (uint32_t j = 0; j < i; ++j) g->loopback |= g->dev[i] == g->dev[j];
    cdb_status rc = group_alloc_slots(g.get(), n_devices);
    if (rc) { cdb_shard_group_destroy(g.release()); return rc; }
    if (n_devices > 1 && !g->loopback) {
        NcclApi *n = nccl_api();
        if (!n) { set_error("libnccl.so.2 not found"); cdb_shard_group_destroy(g.release()); return CDB_NCCL_ERROR; }
        ncclResult_t r = n->CommInitAll(g->comm.data(), (int)n_devices, g->dev.data());
        if (r != ncclSuccess) {
            set_error(std::string("ncclCommInitAll: ") + n->GetErrorString(r));
            for (auto &c : g->comm) c = nullptr;
            cdb_shard_group_destroy(g.release());
            return CDB_NCCL_ERROR;
        }
    }
    *out = g.release();
    return CDB_OK;
}

cdb_status cdb_shard_group_create_rank(const uint8_t *id128, uint32_t world, uint32_t rank, int32_t device, cdb_shard_group **out) {
    CDB_REQUIRE(out && world >= 1 && rank < world && (id128 || world == 1), "bad argument");
    std::unique_ptr<cdb_shard_group> g(new cdb_shard_group());
    g->world = world;
    g->rank0 = rank;
    g->dev.assign(1, device);
    cdb_status rc = group_alloc_slots(g.get(), 1);
    if (rc) { cdb_shard_group_destroy(g.release()); return rc; }
    if (world > 1) {
        NcclApi *n = nccl_api();
        if (!n) { set_error("libnccl.so.2 not found"); cdb_shard_group_destroy(g.release()); return CDB_NCCL_ERROR; }
        ncclUniqueId id;
        memcpy(&id, id128, sizeof(id));
        ncclResult_t r = n->CommInitRank(&g->comm[0], (int)world, id, (int)rank);
        if (r != ncclSuccess) {
            set_error(std::string("ncclCommInitRank: ") + n->GetErrorString(r));
            g->comm[0] = nullptr;
            cdb_shard_group_destroy(g.release());
            return CDB_NCCL_ERROR;
        }
    }
    *out = g.release();
    return CDB_OK;
}

cdb_status cdb_shard_group_destroy(cdb_shard_group *g) {
    if (!g) return CDB_OK;
    NcclApi *n = nccl_api();
    for (size_t i = 0; i < g->dev.size(); ++i) {
        cudaSetDevice(g->dev[i]);
        if (i < g->stream.size() && g->stream[i]) cudaStreamSynchronize(g->stream[i]);
        if (i < g->comm.size() && g->comm[i] && n) n->CommDestroy(g->comm[i]);
        for (auto *v : {&g->gather, &g->q, &g->ids, &g->scores, &g->counts, &g->rows, &g->sel})
            if (i < v->size()) (*v)[i].release();
        if (i < g->ev.size() && g->ev[i]) cudaEventDestroy(g->ev[i]);
        if (i < g->stream.size() && g->stream[i]) cudaStreamDestroy(g->stream[i]);
    }
    delete g;
    return CDB_OK;
}

// [base, base + capacity) of two shards of one local group must not meet: a candidate belongs to exactly one shard
static bool id_ranges_meet(uint32_t b0, uint64_t c0, uint32_t b1, uint64_t c1) { return b0 < b1 + c1 && b1 < b0 + c0; }

// Every local shard gets the same query batch (nq * dim floats) and the merge decodes all their keys with one metric, and
// relies on every key being unique: a shard must agree with every other attached one, whatever the attach order.
cdb_status cdb_shard_group_attach(cdb_shard_group *g, uint32_t local_slot, cdb_index *shard) {
    CDB_REQUIRE(g && shard && local_slot < g->dev.size(), "bad argument");
    CDB_REQUIRE(index_device(shard) == g->dev[local_slot], "the shard lives on another device than the group slot");
    for (size_t j = 0; j < g->dev.size(); ++j) {
        const cdb_index *o = g->shard[j];
        if (!o || j == local_slot) continue;
        CDB_REQUIRE(index_dim(o) == index_dim(shard), "shards differ in dimension");
        CDB_REQUIRE(index_metric(o) == index_metric(shard), "shards differ in metric");
        CDB_REQUIRE(index_storage_type(o) == index_storage_type(shard), "shards differ in storage_type");
        CDB_REQUIRE(!id_ranges_meet(index_id_base(o), index_capacity(o), index_id_base(shard), index_capacity(shard)),
                    "dense shards' id ranges overlap");
    }
    g->shard[local_slot] = shard;
    return CDB_OK;
}

cdb_status cdb_shard_group_attach_sparse(cdb_shard_group *g, uint32_t local_slot, cdb_sparse_index *shard) {
    CDB_REQUIRE(g && shard && local_slot < g->dev.size(), "bad argument");
    CDB_REQUIRE(sparse_index_device(shard) == g->dev[local_slot], "the shard lives on another device than the group slot");
    const float ub = sparse_index_upper_bound(shard);
    for (size_t j = 0; j < g->dev.size(); ++j) {
        const cdb_sparse_index *o = g->sparse[j];
        if (!o || j == local_slot) continue;
        const float oub = sparse_index_upper_bound(o);
        CDB_REQUIRE(sparse_index_bits(o) == sparse_index_bits(shard) && memcmp(&oub, &ub, 4) == 0,
                    "sparse shards differ in quantization_bits or values_upper_bound");
        CDB_REQUIRE(!id_ranges_meet(sparse_index_id_base(o), sparse_index_capacity(o), sparse_index_id_base(shard), sparse_index_capacity(shard)),
                    "sparse shards' id ranges overlap");
    }
    g->sparse[local_slot] = shard;
    return CDB_OK;
}

cdb_status cdb_shard_group_attach_tfidf(cdb_shard_group *g, uint32_t local_slot, cdb_tfidf_index *shard) {
    CDB_REQUIRE(g && shard && local_slot < g->dev.size(), "bad argument");
    CDB_REQUIRE(tfidf_index_device(shard) == g->dev[local_slot], "the shard lives on another device than the group slot");
    for (size_t j = 0; j < g->dev.size(); ++j) {
        const cdb_tfidf_index *o = g->tfidf[j];
        if (!o || j == local_slot) continue;
        CDB_REQUIRE(!id_ranges_meet(tfidf_index_id_base(o), tfidf_index_capacity(o), tfidf_index_id_base(shard), tfidf_index_capacity(shard)),
                    "tf-idf shards' id ranges overlap");
    }
    g->tfidf[local_slot] = shard;
    return CDB_OK;
}

uint32_t cdb_shard_group_world(const cdb_shard_group *g) { return g ? g->world : 0; }

// the stream local slot i works on: the caller's stream in a per-rank group's device form, else the slot's own
static cudaStream_t slot_stream(const cdb_shard_group *g, size_t i, cudaStream_t out_stream) {
    return (g->dev.size() == 1 && out_stream) ? out_stream : g->stream[i];
}

static uint64_t *gather_buf(const cdb_shard_group *g, size_t i) { return reinterpret_cast<uint64_t *>(g->gather[i].p); }

// Rank r's `words` u64 words at gather_buf(slot) + r * words reach every local slot's gather buffer (NCCL all-gather), or,
// in a loopback group, slot 0's buffer only (device copies ordered by events).  Nothing to do in a group of one rank.
static cdb_status group_allgather(cdb_shard_group *g, size_t words, cudaStream_t out_stream) {
    const size_t nl = g->dev.size();
    if (g->world > 1) {
        if (g->loopback) {
            // test mode (a device listed twice): every slot copies its part into slot 0's buffer, ordered by events
            CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
            for (size_t i = 1; i < nl; ++i) {
                CDB_CUDA_TRY(cudaEventRecord(g->ev[i], g->stream[i]));
                CDB_CUDA_TRY(cudaStreamWaitEvent(g->stream[0], g->ev[i], 0));
                CDB_CUDA_TRY(cudaMemcpyAsync(reinterpret_cast<uint64_t *>(g->gather[0].p) + i * words,
                                             reinterpret_cast<uint64_t *>(g->gather[i].p) + i * words, words * 8, cudaMemcpyDeviceToDevice,
                                             g->stream[0]));
            }
        } else {
            NcclApi *n = nccl_api();
            if (!n) { set_error("libnccl.so.2 not found"); return CDB_NCCL_ERROR; }
            CDB_NCCL_TRY(n, n->GroupStart());
            for (size_t i = 0; i < nl; ++i) {
                uint64_t *base = reinterpret_cast<uint64_t *>(g->gather[i].p);
                cudaStream_t s = (nl == 1 && out_stream) ? out_stream : g->stream[i];
                ncclResult_t r = n->AllGather(base + (size_t)(g->rank0 + i) * words, base, words, ncclUint64, g->comm[i], s);
                if (r != ncclSuccess) { n->GroupEnd(); set_error(std::string("ncclAllGather: ") + n->GetErrorString(r)); return CDB_NCCL_ERROR; }
            }
            CDB_NCCL_TRY(n, n->GroupEnd());
        }
    }
    return CDB_OK;
}

// shared memory of merge_gathered_kernel: the world * k keys of one query
constexpr size_t MERGE_SMEM_MAX = 200 * 1024;

// both forms refuse a merge that cannot run before any copy or search is issued; top_k None (merge_runs_kernel, no shared
// memory bound) splits the row width W = k evenly over the ranks
static cdb_status merge_check(const cdb_shard_group *g, const cdb_search_params *p) {
    if (p->flags & CDB_SEARCH_ALL_CANDIDATES) {
        CDB_REQUIRE(p->k % g->world == 0, "CDB_SEARCH_ALL_CANDIDATES: k (the row width) must be a multiple of the world size");
        return CDB_OK;
    }
    CDB_REQUIRE((size_t)g->world * p->k * 8 <= MERGE_SMEM_MAX, "sharded merge: world * k * 8 bytes exceed 200 KB");
    return CDB_OK;
}

// checks that need the shards, under the group's lock and before any copy: every slot has a shard; top_k None: every local
// shard's candidates fit its rank's k / world columns; filtered: every local shard has graph metadata of one md_dims
// (metadata may be attached after cdb_shard_group_attach), returned in *md_dims
static cdb_status shards_check(const cdb_shard_group *g, const cdb_search_params *p, bool filtered, uint32_t *md_dims) {
    for (size_t i = 0; i < g->dev.size(); ++i) {
        CDB_REQUIRE(g->shard[i], "a group slot has no shard attached");
        cdb_status rc;
        if ((p->flags & CDB_SEARCH_ALL_CANDIDATES) && (rc = index_check_all_width(g->shard[i], p->k / g->world))) return rc;
        if (filtered) {
            const uint32_t d = index_md_dims(g->shard[i]);
            CDB_REQUIRE(d, "metadata filters need cdb_index_set_graph_metadata on every shard");
            CDB_REQUIRE(i == 0 || d == *md_dims, "shards differ in md_dims");
            *md_dims = d;
        }
    }
    return CDB_OK;
}

constexpr size_t GROUP_GATHER_BUDGET = 256ull << 20;   // bytes of one chunk's gather buffer; queries are searched in chunks

// queries per chunk when a query takes `per_q` bytes of every rank's gather slot
static uint32_t group_chunk(const cdb_shard_group *g, uint32_t nq, size_t per_q) {
    return (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)nq, 65535, GROUP_GATHER_BUDGET / (g->world * per_q)}));
}

// loopback: a chunk's slots write their gather buffers only after slot 0 copied the previous chunk's out of them
static cdb_status loopback_fence(cdb_shard_group *g) {
    if (!g->loopback) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    CDB_CUDA_TRY(cudaEventRecord(g->ev[0], g->stream[0]));
    for (size_t i = 1; i < g->dev.size(); ++i) CDB_CUDA_TRY(cudaStreamWaitEvent(g->stream[i], g->ev[0], 0));
    return CDB_OK;
}

// local slot i: search its shard into its slot of its gather buffer, then the collective, then (slot 0 / this rank) the merge.
// flt (may be null): slot i's filter CSR on its device.  With k <= 1024 the whole batch is one chunk and merge_gathered_kernel
// keeps the best k; under CDB_SEARCH_ALL_CANDIDATES each rank writes its sorted list into w = k / world columns, the batch is
// searched in chunks whose gather buffer stays within GROUP_GATHER_BUDGET, and merge_runs_kernel concatenates the runs in
// order.  Each shard's reader lock is held while its search is enqueued.
static cdb_status sharded_enqueue(cdb_shard_group *g, uint32_t nq, const cdb_search_params *p, const std::vector<const float *> &d_q,
                                  const std::vector<ShardFilters> *flt, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                  uint8_t *d_err, cudaStream_t out_stream) {
    const size_t nl = g->dev.size();
    const bool all = p->flags & CDB_SEARCH_ALL_CANDIDATES;
    const uint32_t W = p->k, k = all ? W / g->world : W;   // output columns; columns of one rank's slot
    const uint32_t chunk = all ? group_chunk(g, nq, (size_t)k * 8 + 1) : nq;
    cdb_search_params sp = *p;
    sp.k = k;
    cdb_status rc;
    for (size_t i = 0; i < nl; ++i) CDB_REQUIRE(g->shard[i], "a group slot has no shard attached");
    const uint32_t dim = index_dim(g->shard[0]);
    for (size_t i = 0; i < nl; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = g->gather[i].ensure(g->world * slot_words(chunk, k) * 8)) || (rc = g->ids[i].ensure((size_t)chunk * k * 4)) ||
            (rc = g->scores[i].ensure((size_t)chunk * k * 4)) || (rc = g->counts[i].ensure((size_t)chunk * 4)))
            return rc;
    }
    const int metric = index_result_metric(g->shard[0], p->mode);
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        const size_t words = slot_words(c, k);
        if (q0 && (rc = loopback_fence(g))) return rc;
        for (size_t i = 0; i < nl; ++i) {
            CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
            uint64_t *slot = reinterpret_cast<uint64_t *>(g->gather[i].p) + (size_t)(g->rank0 + i) * words;
            ShardFilters f{};
            if (flt) {
                const ShardFilters &a = (*flt)[i];
                f = {a.off ? a.off + q0 : nullptr, a.dims, a.n_rows, a.has ? a.has + q0 : nullptr};
            }
            if ((rc = index_search_device_keys(g->shard[i], d_q[i] + (size_t)q0 * dim, c, &sp, reinterpret_cast<uint32_t *>(g->ids[i].p),
                                               reinterpret_cast<float *>(g->scores[i].p), reinterpret_cast<uint32_t *>(g->counts[i].p),
                                               reinterpret_cast<uint8_t *>(slot + (size_t)c * k), slot, slot_stream(g, i, out_stream),
                                               flt ? &f : nullptr)))
                return rc;
        }
        if ((rc = group_allgather(g, words, out_stream))) return rc;
        // merge on local slot 0
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        const cudaStream_t s0 = slot_stream(g, 0, out_stream);
        const uint64_t *gathered = reinterpret_cast<const uint64_t *>(g->gather[0].p);
        uint32_t *o_ids = d_ids + (size_t)q0 * W;
        float *o_scores = d_scores + (size_t)q0 * W;
        uint32_t *o_counts = d_counts ? d_counts + q0 : nullptr;
        uint8_t *o_err = d_err ? d_err + q0 : nullptr;
        if (all) {
            merge_runs_kernel<<<c, 256, 0, s0>>>(gathered, g->world, c, k, words, metric, o_ids, o_scores, o_counts, o_err);
        } else {
            const size_t smem = (size_t)g->world * k * 8;
            CDB_ALLOW_SMEM(merge_gathered_kernel, smem);
            merge_gathered_kernel<<<c, 128, smem, s0>>>(gathered, g->world, c, k, words, metric, o_ids, o_scores, o_counts, o_err);
        }
        CDB_LAUNCH_CHECK();
    }
    return CDB_OK;
}

cdb_status cdb_search_batch_sharded(cdb_shard_group *g, const float *queries, uint32_t nq, const cdb_search_params *p,
                                    uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(g && p && (queries || !nq) && (out_ids || !nq) && (out_scores || !nq), "null argument");
    if (cdb_status kc = check_search_k(p)) return kc;
    if (!nq) return CDB_OK;
    cdb_status rc = merge_check(g, p);
    if (rc) return rc;
    std::lock_guard<std::mutex> lock(g->mu);
    CDB_REQUIRE(g->shard[0], "a group slot has no shard attached");
    uint32_t md_dims = 0;
    if ((p->flags & CDB_SEARCH_ALL_CANDIDATES) && (rc = shards_check(g, p, false, &md_dims))) return rc;
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{queries, (size_t)nq * index_dim(g->shard[0]) * 4}}, &st)) &&
        !(rc = host_rows(g, nq, p->k, out_ids, out_scores, out_counts, err_flags, &r))) {
        std::vector<const float *> d_q(g->dev.size());
        for (size_t i = 0; i < d_q.size(); ++i) d_q[i] = st.at<float>(i, 0);
        rc = sharded_enqueue(g, nq, p, d_q, nullptr, r.ids, r.scores, r.counts, r.err, nullptr);
    }
    return host_finish(g, rc, &r);
}

cdb_status cdb_search_batch_sharded_device(cdb_shard_group *g, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                           uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts, uint8_t *d_err_flags,
                                           void *stream) {
    CDB_REQUIRE(g && p && (d_queries || !nq) && (d_out_ids || !nq) && (d_out_scores || !nq), "null argument");
    CDB_REQUIRE(g->dev.size() == 1, "the device form serves one-process-per-GPU groups (cdb_shard_group_create_rank)");
    if (cdb_status kc = check_search_k(p)) return kc;
    if (!nq) return CDB_OK;
    cdb_status rc = merge_check(g, p);
    if (rc) return rc;
    std::lock_guard<std::mutex> lock(g->mu);
    uint32_t md_dims = 0;
    if ((p->flags & CDB_SEARCH_ALL_CANDIDATES) && (rc = shards_check(g, p, false, &md_dims))) return rc;
    std::vector<const float *> d_q(1, d_queries);
    return sharded_enqueue(g, nq, p, d_q, nullptr, d_out_ids, d_out_scores, d_out_counts, d_err_flags, (cudaStream_t)stream);
}

// the refusals of cdb_search_batch_filtered[_device] that need no handle, in their order
static cdb_status filtered_params_check(const cdb_search_params *p, const void *offsets, const void *has) {
    CDB_REQUIRE(p->mode == CDB_MODE_HNSW, "metadata filters apply to CDB_MODE_HNSW");
    if (cdb_status kc = check_search_k(p)) return kc;
    CDB_REQUIRE(!has || offsets, "has_filter needs filter_offsets");
    return CDB_OK;
}

cdb_status cdb_search_batch_filtered_sharded(cdb_shard_group *g, const float *queries, uint32_t nq, const cdb_search_params *p,
                                             const uint32_t *filter_offsets, const int8_t *filter_dims, const uint8_t *has_filter,
                                             uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(g && p && (queries || !nq) && (out_ids || !nq) && (out_scores || !nq), "null argument");
    cdb_status rc = filtered_params_check(p, filter_offsets, has_filter);
    if (rc) return rc;
    if (!nq) return CDB_OK;
    if ((rc = merge_check(g, p))) return rc;
    uint32_t total = 0;
    if (has_filter) {
        for (uint32_t q = 0; q < nq; ++q) {
            CDB_REQUIRE(filter_offsets[q] <= filter_offsets[q + 1], "filter_offsets must be non-decreasing");
            CDB_REQUIRE(!has_filter[q] || filter_offsets[q + 1] - filter_offsets[q] <= 4096, "too many filters for one query");
        }
        total = filter_offsets[nq];
        CDB_REQUIRE(filter_dims || !total, "null filter_dims");
    }
    std::lock_guard<std::mutex> lock(g->mu);
    uint32_t md_dims = 0;
    if ((rc = shards_check(g, p, true, &md_dims))) return rc;
    const size_t f = has_filter ? 1 : 0;   // the filter arrays are staged only with has_filter
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{queries, (size_t)nq * index_dim(g->shard[0]) * 4}, {filter_offsets, f * ((size_t)nq + 1) * 4},
                                 {has_filter, f * nq}, {filter_dims, (size_t)total * md_dims}}, &st)) &&
        !(rc = host_rows(g, nq, p->k, out_ids, out_scores, out_counts, err_flags, &r))) {
        std::vector<const float *> d_q(g->dev.size());
        std::vector<ShardFilters> flt(g->dev.size(), ShardFilters{nullptr, nullptr, 0, nullptr});
        for (size_t i = 0; i < d_q.size(); ++i) {
            d_q[i] = st.at<float>(i, 0);
            if (has_filter) flt[i] = {st.at<uint32_t>(i, 1), st.at<int8_t>(i, 3), total, st.at<uint8_t>(i, 2)};
        }
        rc = sharded_enqueue(g, nq, p, d_q, &flt, r.ids, r.scores, r.counts, r.err, nullptr);
    }
    return host_finish(g, rc, &r);
}

cdb_status cdb_search_batch_filtered_sharded_device(cdb_shard_group *g, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                                    const uint32_t *d_filter_offsets, const int8_t *d_filter_dims, uint32_t n_filter_rows,
                                                    const uint8_t *d_has_filter, uint32_t *d_out_ids, float *d_out_scores,
                                                    uint32_t *d_out_counts, uint8_t *d_err_flags, void *stream) {
    CDB_REQUIRE(p, "null params");
    cdb_status rc = filtered_params_check(p, d_filter_offsets, d_has_filter);
    if (rc) return rc;
    CDB_REQUIRE(d_filter_dims || !n_filter_rows, "n_filter_rows > 0 needs filter_dims");
    CDB_REQUIRE(g && (d_queries || !nq) && (d_out_ids || !nq) && (d_out_scores || !nq), "null argument");
    CDB_REQUIRE(g->dev.size() == 1, "the device form serves one-process-per-GPU groups (cdb_shard_group_create_rank)");
    if (!nq) return CDB_OK;
    if ((rc = merge_check(g, p))) return rc;
    std::lock_guard<std::mutex> lock(g->mu);
    uint32_t md_dims = 0;
    if ((rc = shards_check(g, p, true, &md_dims))) return rc;
    std::vector<const float *> d_q(1, d_queries);
    std::vector<ShardFilters> flt(1, ShardFilters{d_filter_offsets, d_filter_dims, n_filter_rows, d_has_filter});
    return sharded_enqueue(g, nq, p, d_q, &flt, d_out_ids, d_out_scores, d_out_counts, d_err_flags, (cudaStream_t)stream);
}

// ---------------------------------------------------------------- sparse and TF-IDF shards

struct SparseQueries {
    const uint64_t *off;
    const uint32_t *dims;
    const float *vals;
};

// Per chunk of queries: phase 1 writes every shard's top m (keys, then counts) into its rank's slot; all-gather #1; the
// group's top m per query (on every local slot, on slot 0 only in loopback).  Without re-rank (m = k) slot 0 sorts those.
// With re-rank, every shard re-ranks the candidates it owns into its rank's slot (0 elsewhere), all-gather #2, and slot 0
// ORs the ranks' lists and sorts them.  The caller holds every local shard's reader lock.
static cdb_status sparse_sharded_enqueue(cdb_shard_group *g, uint32_t nq, const cdb_sparse_search_params *p, uint32_t m,
                                         const std::vector<SparseQueries> &dq, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                         cudaStream_t out_stream) {
    const size_t nl = g->dev.size(), n_sel = g->loopback ? 1 : nl;
    const uint32_t k = p->k, chunk = group_chunk(g, nq, (size_t)m * 8 + 4);
    const size_t cap_words = (size_t)chunk * m + (chunk + 1) / 2;
    cdb_status rc;
    for (size_t i = 0; i < nl; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = g->gather[i].ensure(g->world * cap_words * 8)) || (i < n_sel && (rc = g->sel[i].ensure((size_t)chunk * m * 8 + chunk * 4))))
            return rc;
    }
    const cudaStream_t s0 = slot_stream(g, 0, out_stream);
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        const size_t words = (size_t)c * m + (c + 1) / 2;
        if (q0 && (rc = loopback_fence(g))) return rc;
        for (size_t i = 0; i < nl; ++i) {
            CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
            uint64_t *slot = gather_buf(g, i) + (g->rank0 + i) * words;
            if ((rc = sparse_shard_select(g->sparse[i], dq[i].off + q0, dq[i].dims, dq[i].vals, c, p, m, slot,
                                          reinterpret_cast<uint32_t *>(slot + (size_t)c * m), slot_stream(g, i, out_stream))))
                return rc;
        }
        if ((rc = group_allgather(g, words, out_stream))) return rc;
        auto sel_keys = [&](size_t i) { return reinterpret_cast<uint64_t *>(g->sel[i].p); };
        auto sel_cnt = [&](size_t i) { return reinterpret_cast<uint32_t *>(sel_keys(i) + (size_t)c * m); };
        for (size_t i = 0; i < n_sel; ++i) {
            CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
            if ((rc = sparse_group_select(gather_buf(g, i), words, g->world, c, m, sel_keys(i), sel_cnt(i), slot_stream(g, i, out_stream))))
                return rc;
        }
        if (p->rerank) {
            // loopback: every shard re-ranks on slot 0's stream from slot 0's list straight into slot 0's gather buffer
            for (size_t i = 0; i < nl; ++i) {
                const size_t j = g->loopback ? 0 : i;
                CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
                if ((rc = sparse_shard_rerank(g->sparse[i], dq[i].off + q0, dq[i].dims, dq[i].vals, c, m, sel_keys(j), sel_cnt(j),
                                              gather_buf(g, j) + (g->rank0 + i) * words, slot_stream(g, j, out_stream))))
                    return rc;
            }
            if (!g->loopback && (rc = group_allgather(g, words, out_stream))) return rc;
        }
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        if ((rc = sparse_group_finalize(gather_buf(g, 0), words, g->world, c, m, k, p->rerank ? 1 : 0, sel_keys(0), sel_cnt(0),
                                        d_ids + (size_t)q0 * k, d_scores + (size_t)q0 * k, d_counts + q0, s0)))
            return rc;
    }
    return CDB_OK;
}

// every local slot needs a sparse shard (both forms refuse before any device work: parameters, arguments, slots)
static cdb_status sparse_sharded_slots(const cdb_shard_group *g) {
    for (size_t i = 0; i < g->dev.size(); ++i) CDB_REQUIRE(g->sparse[i], "a group slot has no sparse shard attached");
    return CDB_OK;
}

// a sparse query CSR staged as arrays j, j + 1, j + 2 (offsets, dims, values), on every local slot
static std::vector<SparseQueries> staged_sparse(const Staged &st, size_t j) {
    std::vector<SparseQueries> q(st.base.size());
    for (size_t i = 0; i < q.size(); ++i) q[i] = {st.at<uint64_t>(i, j), st.at<uint32_t>(i, j + 1), st.at<float>(i, j + 2)};
    return q;
}

cdb_status cdb_sparse_search_batch_sharded(cdb_shard_group *g, const uint64_t *q_offsets, const uint32_t *q_dims, const float *q_values,
                                           uint32_t nq, const cdb_sparse_search_params *p, uint32_t *out_ids, float *out_scores,
                                           uint32_t *out_counts) {
    uint32_t m = 0;
    cdb_status rc = sparse_check_params(p, &m);
    if (rc) return rc;
    CDB_REQUIRE(g && (out_ids || !nq) && (out_scores || !nq) && (out_counts || !nq), "null argument");
    if ((rc = sparse_sharded_slots(g))) return rc;
    if (!nq) return CDB_OK;
    if ((rc = check_csr(q_offsets, nq, "q_offsets"))) return rc;
    const uint64_t nqp = q_offsets[nq];
    CDB_REQUIRE((q_dims && q_values) || !nqp, "null query pairs");
    std::lock_guard<std::mutex> lock(g->mu);
    const size_t nl = g->dev.size();
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) locks.emplace_back(sparse_index_mutex(g->sparse[i]));
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{q_offsets, ((size_t)nq + 1) * 8}, {q_dims, nqp * 4}, {q_values, nqp * 4}}, &st)) &&
        !(rc = host_rows(g, nq, p->k, out_ids, out_scores, out_counts, nullptr, &r)))
        rc = sparse_sharded_enqueue(g, nq, p, m, staged_sparse(st, 0), r.ids, r.scores, r.counts, nullptr);
    return host_finish(g, rc, &r);
}

cdb_status cdb_sparse_search_batch_sharded_device(cdb_shard_group *g, const uint64_t *d_q_offsets, const uint32_t *d_q_dims,
                                                  const float *d_q_values, uint32_t nq, const cdb_sparse_search_params *p, uint32_t *d_ids,
                                                  float *d_scores, uint32_t *d_counts, void *stream) {
    uint32_t m = 0;
    cdb_status rc = sparse_check_params(p, &m);
    if (rc) return rc;
    CDB_REQUIRE(g && (d_q_offsets || !nq) && (d_ids || !nq) && (d_scores || !nq) && (d_counts || !nq), "null argument");
    CDB_REQUIRE(g->dev.size() == 1, "the device form serves one-process-per-GPU groups (cdb_shard_group_create_rank)");
    if ((rc = sparse_sharded_slots(g))) return rc;
    if (!nq) return CDB_OK;
    std::lock_guard<std::mutex> lock(g->mu);
    std::shared_lock<std::shared_mutex> shard_lock(sparse_index_mutex(g->sparse[0]));
    std::vector<SparseQueries> dq(1, SparseQueries{d_q_offsets, d_q_dims, d_q_values});
    return sparse_sharded_enqueue(g, nq, p, m, dq, d_ids, d_scores, d_counts, (cudaStream_t)stream);
}

// ---------------------------------------------------------------- top_k None over the sparse shards (DESIGN.md section 8f)

// The key exchange of one scoring chunk of c queries, from the all-gathered counts cnt[r * c + qi] alone, so every rank
// derives the same sub-batches: consecutive queries [b[s], b[s+1]) whose largest rank total `words` keeps world * words * 8
// bytes within GROUP_GATHER_BUDGET (a sub-batch holds at least one query, which may exceed it).  Sub-batches without a key
// are dropped: they need no exchange.
struct KeyBatch {
    uint32_t a, b;   // queries [a, b) of the chunk
    size_t words;    // keys of the largest rank
};
static std::vector<KeyBatch> key_batches(const std::vector<uint32_t> &cnt, uint32_t world, uint32_t c) {
    std::vector<KeyBatch> out;
    std::vector<uint64_t> tot(world);
    const uint64_t cap = GROUP_GATHER_BUDGET / (8ull * world);
    for (uint32_t a = 0; a < c;) {
        std::fill(tot.begin(), tot.end(), 0);
        uint64_t words = 0;
        uint32_t b = a;
        for (; b < c; ++b) {
            uint64_t w = 0;
            for (uint32_t r = 0; r < world; ++r) w = std::max(w, tot[r] + cnt[(size_t)r * c + b]);
            if (b > a && w > cap) break;
            for (uint32_t r = 0; r < world; ++r) tot[r] += cnt[(size_t)r * c + b];
            words = w;
        }
        if (words) out.push_back({a, b, (size_t)words});
        a = b;
    }
    return out;
}

// Under g->mu and every local shard's reader lock.  Plan (per-rank groups: one all-gather of each rank's tiles and live
// rows), then per scoring chunk: every local shard's device half into its own scratch; an all-gather of the per-query
// counts; per key sub-batch, every rank's sorted keys into its slot, an all-gather, and the merge on local slot 0, copied
// into r.  Every rank issues the same collectives: the chunk comes from group-wide maxima, the sub-batches from the
// gathered counts.
static cdb_status sparse_all_sharded_run(cdb_shard_group *g, const std::vector<SparseQueries> &dq, uint32_t nq,
                                         const cdb_sparse_search_params *p, cdb_sparse_results *r, std::vector<SparseAllScratch> &sc) {
    const size_t nl = g->dev.size();
    const uint32_t world = g->world;
    cdb_status rc;
    // plan: [tiles, live rows] of every rank
    std::vector<uint64_t> bounds(2 * (size_t)world, 0);
    for (size_t i = 0; i < nl; ++i) sparse_index_all_bounds(g->sparse[i], &bounds[2 * (g->rank0 + i)], &bounds[2 * (g->rank0 + i) + 1]);
    if (nl < world) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        if ((rc = g->gather[0].ensure((size_t)world * 16))) return rc;
        CDB_CUDA_TRY(cudaMemcpyAsync(gather_buf(g, 0) + 2 * g->rank0, &bounds[2 * g->rank0], 16, cudaMemcpyHostToDevice, g->stream[0]));
        if ((rc = group_allgather(g, 2, nullptr))) return rc;
        CDB_CUDA_TRY(cudaMemcpyAsync(bounds.data(), gather_buf(g, 0), (size_t)world * 16, cudaMemcpyDeviceToHost, g->stream[0]));
        CDB_CUDA_TRY(cudaStreamSynchronize(g->stream[0]));
    }
    uint64_t max_tiles = 0, max_live = 0, sum_live = 0;
    for (uint32_t k = 0; k < world; ++k) {
        max_tiles = std::max(max_tiles, bounds[2 * k]);
        max_live = std::max(max_live, bounds[2 * k + 1]);
        sum_live += bounds[2 * k + 1];
    }
    CDB_REQUIRE(sum_live < (1ull << 31), "top_k None: a shard group with 2^31 live rows or more");
    if (!max_tiles || !max_live) return CDB_OK;   // no rank has a candidate: r holds nq empty queries
    const uint32_t chunk = sparse_all_chunk(nq, max_tiles, max_live);
    for (size_t i = 0; i < nl; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = sparse_all_alloc(g->sparse[i], chunk, &sc[i], g->stream[i]))) return rc;
    }
    const cudaStream_t s0 = g->stream[0];
    std::vector<uint32_t> cnt, pre;
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        const size_t cw = ((size_t)c + 1) / 2;   // u64 words of c u32 counts
        if (q0 && (rc = loopback_fence(g))) return rc;
        for (size_t i = 0; i < nl; ++i) {
            CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
            if ((rc = sparse_all_keys(g->sparse[i], dq[i].off, dq[i].dims, dq[i].vals, p, q0, c, &sc[i], g->stream[i]))) return rc;
            std::vector<uint32_t> &seg = sc[i].seg_h;
            for (uint32_t qi = 0; qi < c; ++qi) seg[qi] = seg[qi + 1] - seg[qi];   // counts; seg[c] stays the total
            if ((rc = g->gather[i].ensure((size_t)world * cw * 8))) return rc;
            CDB_CUDA_TRY(cudaMemcpyAsync(gather_buf(g, i) + (g->rank0 + i) * cw, seg.data(), (size_t)c * 4, cudaMemcpyHostToDevice, g->stream[i]));
        }
        if ((rc = group_allgather(g, cw, nullptr))) return rc;
        std::vector<uint32_t> all(world * cw * 2);
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        CDB_CUDA_TRY(cudaMemcpyAsync(all.data(), gather_buf(g, 0), all.size() * 4, cudaMemcpyDeviceToHost, s0));
        CDB_CUDA_TRY(cudaStreamSynchronize(s0));
        cnt.assign((size_t)world * c, 0);
        for (uint32_t k = 0; k < world; ++k) std::copy(&all[k * cw * 2], &all[k * cw * 2] + c, &cnt[(size_t)k * c]);
        for (uint32_t qi = 0; qi < c; ++qi) {
            uint64_t t = 0;
            for (uint32_t k = 0; k < world; ++k) t += cnt[(size_t)k * c + qi];
            r->off[(size_t)q0 + qi + 1] = r->off[(size_t)q0 + qi] + t;
        }
        r->ids.resize(r->off[(size_t)q0 + c]);
        r->scores.resize(r->off[(size_t)q0 + c]);
        // every local shard's keys of query qi start at key_beg[i][qi] of its sorted run
        std::vector<std::vector<uint32_t>> key_beg(nl, std::vector<uint32_t>((size_t)c + 1, 0));
        for (size_t i = 0; i < nl; ++i)
            for (uint32_t qi = 0; qi < c; ++qi) key_beg[i][qi + 1] = key_beg[i][qi] + sc[i].seg_h[qi];
        for (const KeyBatch &kb : key_batches(cnt, world, c)) {
            const uint32_t nb = kb.b - kb.a;
            if ((rc = loopback_fence(g))) return rc;
            for (size_t i = 0; i < nl; ++i) {
                CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
                if ((rc = g->gather[i].ensure((size_t)world * kb.words * 8))) return rc;
                const uint32_t b = key_beg[i][kb.a], e = key_beg[i][kb.b];
                if (e > b)
                    CDB_CUDA_TRY(cudaMemcpyAsync(gather_buf(g, i) + (g->rank0 + i) * kb.words, sc[i].keys + b, (size_t)(e - b) * 8,
                                                 cudaMemcpyDeviceToDevice, g->stream[i]));
            }
            if ((rc = group_allgather(g, kb.words, nullptr))) return rc;
            pre.assign((size_t)world * (nb + 1), 0);
            uint64_t n = 0;
            for (uint32_t k = 0; k < world; ++k) {
                uint32_t *P = &pre[(size_t)k * (nb + 1)];
                for (uint32_t j = 0; j < nb; ++j) P[j + 1] = P[j] + cnt[(size_t)k * c + kb.a + j];
                n += P[nb];
            }
            CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
            if ((rc = g->sel[0].ensure(pre.size() * 4)) || (rc = g->ids[0].ensure(n * 4)) || (rc = g->scores[0].ensure(n * 4))) return rc;
            uint32_t *d_pre = reinterpret_cast<uint32_t *>(g->sel[0].p);
            uint32_t *d_ids = reinterpret_cast<uint32_t *>(g->ids[0].p);
            float *d_scores = reinterpret_cast<float *>(g->scores[0].p);
            CDB_CUDA_TRY(cudaMemcpyAsync(d_pre, pre.data(), pre.size() * 4, cudaMemcpyHostToDevice, s0));
            if ((rc = sparse_group_merge_all(gather_buf(g, 0), kb.words, world, d_pre, nb, (uint32_t)n, p->rerank ? 1 : 0, d_ids, d_scores, s0)))
                return rc;
            const uint64_t base = r->off[(size_t)q0 + kb.a];
            CDB_CUDA_TRY(cudaMemcpyAsync(r->ids.data() + base, d_ids, n * 4, cudaMemcpyDeviceToHost, s0));
            CDB_CUDA_TRY(cudaMemcpyAsync(r->scores.data() + base, d_scores, n * 4, cudaMemcpyDeviceToHost, s0));
            CDB_CUDA_TRY(cudaStreamSynchronize(s0));
        }
    }
    return CDB_OK;
}

cdb_status cdb_sparse_search_batch_all_sharded(cdb_shard_group *g, const uint64_t *q_offsets, const uint32_t *q_dims, const float *q_values,
                                               uint32_t nq, const cdb_sparse_search_params *p, cdb_sparse_results **out) {
    CDB_REQUIRE(g && p && out, "null argument");
    *out = nullptr;
    CDB_REQUIRE(p->k == 0, "cdb_sparse_search_batch_all_sharded takes k = 0 (top_k None)");
    if (nq) {
        cdb_status rc = check_csr(q_offsets, nq, "q_offsets");
        if (rc) return rc;
        CDB_REQUIRE((q_dims && q_values) || !q_offsets[nq], "null query pairs");
    }
    if (cdb_status rc = sparse_sharded_slots(g)) return rc;
    std::unique_ptr<cdb_sparse_results> r(new (std::nothrow) cdb_sparse_results());
    CDB_REQUIRE(r, "out of host memory");
    cdb_status rc = CDB_OK;
    try {
        r->off.assign((size_t)nq + 1, 0);
    } catch (const std::bad_alloc &) {
        set_error("top_k None: host allocation of the results failed");
        return CDB_CUDA_ERROR;
    }
    if (!nq) {   // every rank passes the same n_queries: none runs a collective
        *out = r.release();
        return CDB_OK;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    const size_t nl = g->dev.size();
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) locks.emplace_back(sparse_index_mutex(g->sparse[i]));
    const uint64_t nqp = q_offsets[nq];
    std::vector<SparseAllScratch> sc(nl);
    Staged st;
    rc = stage_queries(g, {{q_offsets, ((size_t)nq + 1) * 8}, {q_dims, nqp * 4}, {q_values, nqp * 4}}, &st);
    if (!rc) {
        try {
            rc = sparse_all_sharded_run(g, staged_sparse(st, 0), nq, p, r.get(), sc);
        } catch (const std::bad_alloc &) {
            set_error("top_k None: host allocation of the results failed");
            rc = CDB_CUDA_ERROR;
        }
    }
    for (size_t i = 0; i < nl; ++i) {   // scratch is freed behind its last use
        cudaSetDevice(g->dev[i]);
        sparse_all_free(&sc[i], g->stream[i]);
    }
    if ((rc = host_finish(g, rc, nullptr))) return rc;
    *out = r.release();
    return CDB_OK;
}

// ---------------------------------------------------------------- TF-IDF shards (DESIGN.md section 8f)

// one local slot's query CSR on its device: offsets index the batch's whole hash array
struct TfQueries {
    const uint64_t *off;
    const uint32_t *hashes;
};

// a TF-IDF query CSR staged as arrays j, j + 1 (offsets, hashes), on every local slot
static std::vector<TfQueries> staged_tfidf(const Staged &st, size_t j) {
    std::vector<TfQueries> q(st.base.size());
    for (size_t i = 0; i < q.size(); ++i) q[i] = {st.at<uint64_t>(i, j), st.at<uint32_t>(i, j + 1)};
    return q;
}

// The TF-IDF plan's first step, once per batch: the group's idf of its nqh query terms.  Every local slot writes its
// shard's [N, df of every query term] (u32) into its rank's slot of its gather buffer; one all-gather; then N and each df
// are summed over the ranks (u32, wrapping) and bm25_idf of every term lands in scratch allocated on the slot's stream:
// every local slot's from its own gather buffer into (*idf)[i], or, in loopback, where only slot 0's buffer is complete,
// slot 0's into (*idf)[0], which every slot reads behind the fence at the end.  The gather buffers are sized for the
// scoring of nq queries as well.  tfidf_idf_free releases the scratch behind its last reader.
static cdb_status tfidf_idf_enqueue(cdb_shard_group *g, const std::vector<TfQueries> &tq, uint32_t nq, uint64_t nqh,
                                    std::vector<float *> *idf, cudaStream_t out_stream) {
    const size_t nl = g->dev.size(), words = (nqh + 2) / 2;   // one rank's [N, df...] in u64 words
    const size_t score_words = (size_t)group_chunk(g, nq, 512 * 8) * 512;
    cdb_status rc;
    idf->assign(g->loopback ? 1 : nl, nullptr);
    for (size_t i = 0; i < nl; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = g->gather[i].ensure(g->world * std::max(words, score_words) * 8))) return rc;
    }
    for (size_t i = 0; i < nl; ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        const cudaStream_t s = slot_stream(g, i, out_stream);
        if (i < idf->size() && nqh) CDB_CUDA_TRY(cudaMallocAsync(&(*idf)[i], nqh * 4, s));
        if ((rc = tfidf_shard_stats(g->tfidf[i], tq[i].hashes, nqh, reinterpret_cast<uint32_t *>(gather_buf(g, i) + (g->rank0 + i) * words), s)))
            return rc;
    }
    if ((rc = group_allgather(g, words, out_stream))) return rc;
    for (size_t i = 0; i < idf->size(); ++i) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
        if ((rc = tfidf_group_idf(gather_buf(g, i), words, g->world, nqh, (*idf)[i], slot_stream(g, i, out_stream)))) return rc;
    }
    return loopback_fence(g);
}

// on the stream that allocated it: every reader's last work is on it, or (loopback) joined it in the last all-gather
static void tfidf_idf_free(cdb_shard_group *g, const std::vector<float *> &idf, cudaStream_t out_stream) {
    for (size_t i = 0; i < idf.size(); ++i)
        if (idf[i]) {
            cudaSetDevice(g->dev[i]);
            cudaFreeAsync(idf[i], slot_stream(g, i, out_stream));
        }
}

// The TF-IDF plan's second step, for queries [q0, q0 + c) of the batch under its idf, per group chunk: every local shard
// writes all 512 bucket winners per query into its rank's slot; one all-gather; slot 0 takes the best of the ranks per
// bucket and sorts them into ids / scores [c][tfidf_out_cols(k)] and counts [c] on slot 0.
static cdb_status tfidf_sharded_enqueue(cdb_shard_group *g, const std::vector<TfQueries> &tq, uint64_t nqh, const std::vector<float *> &idf,
                                        uint32_t q0, uint32_t c, uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                        cudaStream_t out_stream) {
    const uint32_t kout = tfidf_out_cols(k), chunk = group_chunk(g, c, 512 * 8);
    cdb_status rc;
    for (uint32_t a = 0; a < c; a += chunk) {
        const uint32_t n = std::min(chunk, c - a);
        const size_t words = (size_t)n * 512;
        if (a && (rc = loopback_fence(g))) return rc;
        for (size_t i = 0; i < g->dev.size(); ++i) {
            CDB_CUDA_TRY(cudaSetDevice(g->dev[i]));
            if ((rc = tfidf_shard_winners(g->tfidf[i], tq[i].off + q0 + a, tq[i].hashes, nqh, idf[g->loopback ? 0 : i], n,
                                          reinterpret_cast<uint2 *>(gather_buf(g, i) + (g->rank0 + i) * words), slot_stream(g, i, out_stream))))
                return rc;
        }
        if ((rc = group_allgather(g, words, out_stream))) return rc;
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        if ((rc = tfidf_group_finalize(gather_buf(g, 0), words, g->world, n, k, d_ids + (size_t)a * kout, d_scores + (size_t)a * kout,
                                       d_counts + a, slot_stream(g, 0, out_stream))))
            return rc;
    }
    return CDB_OK;
}

// Both steps over a whole batch, on the group's streams (or out_stream, see slot_stream).  The caller holds g->mu and every
// local shard's reader lock through the enqueue.
static cdb_status tfidf_sharded_search(cdb_shard_group *g, const std::vector<TfQueries> &tq, uint32_t nq, uint64_t nqh, uint32_t k,
                                       uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t out_stream) {
    std::vector<float *> idf;
    cdb_status rc = tfidf_idf_enqueue(g, tq, nq, nqh, &idf, out_stream);
    if (!rc) rc = tfidf_sharded_enqueue(g, tq, nqh, idf, 0, nq, k, d_ids, d_scores, d_counts, out_stream);
    tfidf_idf_free(g, idf, out_stream);
    return rc;
}

cdb_status cdb_tfidf_search_batch_sharded(cdb_shard_group *g, const uint64_t *q_offsets, const uint32_t *q_hashes, uint32_t nq, uint32_t k,
                                          uint32_t *out_ids, float *out_scores, uint32_t *out_counts) {
    CDB_REQUIRE(g && (out_ids || !nq) && (out_scores || !nq) && (out_counts || !nq), "null argument");
    const size_t nl = g->dev.size();
    for (size_t i = 0; i < nl; ++i) CDB_REQUIRE(g->tfidf[i], "a group slot has no tf-idf shard attached");
    if (!nq) return CDB_OK;
    cdb_status rc = check_csr(q_offsets, nq, "q_offsets");
    if (rc) return rc;
    const uint64_t nqh = q_offsets[nq];
    CDB_REQUIRE(q_hashes || !nqh, "null query hashes");
    CDB_REQUIRE(nqh < (1ull << 31), "a batch of 2^31 query terms or more");
    std::lock_guard<std::mutex> lock(g->mu);
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) locks.emplace_back(tfidf_index_mutex(g->tfidf[i]));
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{q_offsets, ((size_t)nq + 1) * 8}, {q_hashes, nqh * 4}}, &st)) &&
        !(rc = host_rows(g, nq, tfidf_out_cols(k), out_ids, out_scores, out_counts, nullptr, &r)))
        rc = tfidf_sharded_search(g, staged_tfidf(st, 0), nq, nqh, k, r.ids, r.scores, r.counts, nullptr);
    return host_finish(g, rc, &r);
}

cdb_status cdb_tfidf_search_batch_sharded_device(cdb_shard_group *g, const uint64_t *d_q_offsets, const uint32_t *d_q_hashes, uint32_t nq,
                                                 uint64_t n_query_hashes, uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                                 void *stream) {
    CDB_REQUIRE(g && (d_q_offsets || !nq) && (d_ids || !nq) && (d_scores || !nq) && (d_counts || !nq), "null argument");
    CDB_REQUIRE(d_q_hashes || !nq || !n_query_hashes, "null query hashes");
    CDB_REQUIRE(n_query_hashes < (1ull << 31), "a batch of 2^31 query terms or more");
    const size_t nl = g->dev.size();
    for (size_t i = 1; i < nl; ++i)
        CDB_REQUIRE(g->dev[i] == g->dev[0], "the device form serves groups whose local slots share one device (per-rank, one-slot or loopback)");
    for (size_t i = 0; i < nl; ++i) CDB_REQUIRE(g->tfidf[i], "a group slot has no tf-idf shard attached");
    if (!nq) return CDB_OK;
    std::lock_guard<std::mutex> lock(g->mu);
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) locks.emplace_back(tfidf_index_mutex(g->tfidf[i]));
    // every slot's work follows what the caller's stream held, and the caller's later work follows slot 0's, which joined
    // every slot's last work (collective or loopback copy)
    const cudaStream_t out = (cudaStream_t)stream, s0 = slot_stream(g, 0, out);
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    bool fenced = false;
    for (size_t i = 0; i < nl; ++i) {
        const cudaStream_t si = slot_stream(g, i, out);
        if (si == out) continue;
        if (!fenced) CDB_CUDA_TRY(cudaEventRecord(g->ev[0], out));
        fenced = true;
        CDB_CUDA_TRY(cudaStreamWaitEvent(si, g->ev[0], 0));
    }
    const cdb_status rc = tfidf_sharded_search(g, std::vector<TfQueries>(nl, TfQueries{d_q_offsets, d_q_hashes}), nq, n_query_hashes, k, d_ids,
                                               d_scores, d_counts, out);
    if (s0 != out) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        CDB_CUDA_TRY(cudaEventRecord(g->ev[0], s0));
        CDB_CUDA_TRY(cudaStreamWaitEvent(out, g->ev[0], 0));
    }
    return rc;
}

// ---------------------------------------------------------------- hybrid search over the group (DESIGN.md section 8h)

enum HybSource { HYB_DENSE = 0, HYB_SPARSE = 1, HYB_TFIDF = 2 };

struct HybPlan {
    bool use[3] = {false, false, false};   // the sources searched, always in the order dense, sparse, TF-IDF
    uint32_t nq[3] = {0, 0, 0};            // each searched source's queries
    uint32_t ld[3] = {0, 0, 0};            // columns of each source's intermediate list
    cdb_search_params dense;               // at k = 3 * top_k
    cdb_sparse_search_params sparse;
    uint32_t m = 0;                        // the sparse search's candidates per query
    bool md = false;                       // the dense shards have graph metadata: the filtered path, no filter
};

// the refusals after the source list: the sparse rerank bound, then the sub-searches' own parameter checks at k = 3 * top_k
static cdb_status hyb_params(const cdb_search_params &dense, const cdb_sparse_search_params &sparse, uint32_t top_k, HybPlan *p) {
    const uint32_t k3 = 3 * top_k;
    for (int j = 0; j < 3; ++j) p->ld[j] = j == HYB_TFIDF ? std::min(k3, 512u) : k3;
    if (p->use[HYB_SPARSE] && sparse.rerank)
        CDB_REQUIRE(sparse.reranking_factor >= 1 && (uint64_t)k3 * sparse.reranking_factor <= 5120,
                    "3 * top_k * reranking_factor must be in 1..5120");
    p->dense = dense;
    p->dense.k = k3;
    p->sparse = sparse;
    p->sparse.k = k3;
    if (top_k && p->use[HYB_DENSE])
        if (cdb_status rc = check_search_k(&p->dense)) return rc;
    if (top_k && p->use[HYB_SPARSE])
        if (cdb_status rc = sparse_check_params(&p->sparse, &p->m)) return rc;
    return CDB_OK;
}

// the refusals that need no group, in the order of cdb_hybrid_search_batch's (make_plan in hybrid.cu), then hyb_params
static cdb_status hyb_plan(const cdb_hybrid_group_sources *h, uint32_t nq, uint32_t top_k, HybPlan *p) {
    CDB_REQUIRE(h, "null sources");
    CDB_REQUIRE(top_k <= HYB_MAX_TOP_K, "top_k must be <= 341 (each sub-search takes 3 * top_k <= 1024)");
    CDB_REQUIRE((h->use_dense != 0) + (h->use_sparse != 0) + (h->use_tfidf != 0) == 2, "a hybrid search takes exactly two sources");
    CDB_REQUIRE(!h->use_dense || !(h->dense_params.flags & CDB_SEARCH_ALL_CANDIDATES),
                "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k");
    p->use[HYB_DENSE] = h->use_dense;
    p->use[HYB_SPARSE] = h->use_sparse;
    p->use[HYB_TFIDF] = h->use_tfidf;
    for (int j = 0; j < 3; ++j) p->nq[j] = p->use[j] ? nq : 0;
    CDB_REQUIRE(!h->use_dense || h->dense_queries || !nq, "null dense queries");
    CDB_REQUIRE(!h->use_sparse || h->sparse_offsets || !nq, "null sparse query offsets");
    CDB_REQUIRE(!h->use_tfidf || h->tfidf_offsets || !nq, "null tf-idf query offsets");
    return hyb_params(h->dense_params, h->sparse_params, top_k, p);
}

// a mixed batch's refusals that need no group, in the order of cdb_hybrid_search_batch_mixed's: the sources searched are
// those with queries
static cdb_status hyb_mixed_plan(const cdb_hybrid_group_mixed_sources *h, uint32_t nq, uint32_t top_k, HybPlan *p) {
    CDB_REQUIRE(h, "null sources");
    CDB_REQUIRE(top_k <= HYB_MAX_TOP_K, "top_k must be <= 341 (each sub-search takes 3 * top_k <= 1024)");
    const uint32_t n_src[3] = {h->n_dense, h->n_sparse, h->n_tfidf};
    if (cdb_status rc = check_kinds(h->kinds, nq, n_src)) return rc;
    CDB_REQUIRE(!h->n_dense || !(h->dense_params.flags & CDB_SEARCH_ALL_CANDIDATES),
                "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k");
    for (int j = 0; j < 3; ++j) {
        p->use[j] = n_src[j] != 0;
        p->nq[j] = n_src[j];
    }
    CDB_REQUIRE(!h->n_dense || h->dense_queries, "null dense queries");
    CDB_REQUIRE(!h->n_sparse || h->sparse_offsets, "null sparse query offsets");
    CDB_REQUIRE(!h->n_tfidf || h->tfidf_offsets, "null tf-idf query offsets");
    return hyb_params(h->dense_params, h->sparse_params, top_k, p);
}

// the host form's query CSRs, before the group is locked: n_sp / n_tf queries of each searched text source
static cdb_status hyb_check_csr(const uint64_t *sp_off, const uint32_t *sp_dims, const float *sp_vals, uint32_t n_sp,
                                const uint64_t *tf_off, const uint32_t *tf_hashes, uint32_t n_tf) {
    cdb_status rc;
    if (n_sp) {
        if ((rc = check_csr(sp_off, n_sp, "sparse_offsets"))) return rc;
        CDB_REQUIRE((sp_dims && sp_vals) || !sp_off[n_sp], "null sparse query pairs");
    }
    if (n_tf) {
        if ((rc = check_csr(tf_off, n_tf, "tfidf_offsets"))) return rc;
        CDB_REQUIRE(tf_hashes || !tf_off[n_tf], "null tf-idf query hashes");
        CDB_REQUIRE(tf_off[n_tf] < (1ull << 31), "a batch of 2^31 query terms or more");
    }
    return CDB_OK;
}

// under g->mu, before any copy: every local slot has a shard of each searched kind; the dense shards all have graph metadata
// (of one md_dims; HNSW only) or none has; the dense merge fits
static cdb_status hyb_group_check(const cdb_shard_group *g, HybPlan *p) {
    const size_t nl = g->dev.size();
    for (size_t i = 0; i < nl; ++i) {
        CDB_REQUIRE(!p->use[HYB_DENSE] || g->shard[i], "a group slot has no shard attached");
        CDB_REQUIRE(!p->use[HYB_SPARSE] || g->sparse[i], "a group slot has no sparse shard attached");
        CDB_REQUIRE(!p->use[HYB_TFIDF] || g->tfidf[i], "a group slot has no tf-idf shard attached");
    }
    if (!p->use[HYB_DENSE]) return CDB_OK;
    size_t with_md = 0;
    for (size_t i = 0; i < nl; ++i) with_md += index_md_dims(g->shard[i]) != 0;
    CDB_REQUIRE(with_md == 0 || with_md == nl,
                "hybrid search: some local dense shards have graph metadata and some do not (the dense side takes one path)");
    p->md = with_md != 0;
    CDB_REQUIRE(!p->md || p->dense.mode == CDB_MODE_HNSW, "dense shards with graph metadata search in CDB_MODE_HNSW");
    uint32_t md_dims = 0;
    cdb_status rc = shards_check(g, &p->dense, p->md, &md_dims);
    if (rc) return rc;
    return merge_check(g, &p->dense);
}

// The sub-searches and the fusion, per chunk of request positions, under g->mu and every searched text shard's reader lock.
// dq / sq / tq: each local slot's dense queries, sparse CSR and TF-IDF CSR on its device (nqh: the TF-IDF batch's term
// count).  A pair (kinds null) searches both sources over the chunk's queries and fuses them row by row, the dense search
// writing d_err; a mixed batch (kinds [nq], host) searches each source over its range of the chunk and fuses each kind
// present through its row maps, which scatter the dense error bytes.  A TF-IDF source's idf step runs once, over its whole
// batch, before the chunks.  The sub-searches run one after the other in the order dense, sparse, TF-IDF, each on the
// streams its public entry point uses, so every rank issues the same collectives in the same order, and a source with no
// queries in a chunk issues none; each one's merged list lands in this call's scratch on slot 0, where the fusion writes
// rows q0.. of the output.  Nothing here waits for the device.
static cdb_status hybrid_group_run(cdb_shard_group *g, const HybPlan &p, const uint8_t *kinds, uint32_t nq, uint32_t top_k,
                                   float fusion_k, uint32_t dense_id_stride, const std::vector<const float *> &dq,
                                   const std::vector<SparseQueries> &sq, const std::vector<TfQueries> &tq, uint64_t nqh, uint32_t *d_ids,
                                   float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t out_stream) {
    const size_t nl = g->dev.size();
    const uint32_t k3 = 3 * top_k, ld_out = 6 * top_k;
    // bytes of one request position: ids and scores of its two lists, two counts (a mixed batch: the widest kind present,
    // and the dense error byte)
    size_t per_q = 0;
    if (!kinds) {
        for (int j = 0; j < 3; ++j) per_q += p.use[j] ? (size_t)p.ld[j] * 8 + 4 : 0;
    } else {
        bool present[3] = {false, false, false};
        for (uint32_t q = 0; q < nq; ++q) present[kinds[q]] = true;
        for (int kd = 0; kd < 3; ++kd)
            if (present[kd]) per_q = std::max(per_q, ((size_t)p.ld[HYB_KIND_SRC[kd][0]] + p.ld[HYB_KIND_SRC[kd][1]]) * 8 + 9);
    }
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(nq, GROUP_GATHER_BUDGET / per_q));
    std::vector<MixedChunk> chunks;
    std::vector<uint32_t> maps;
    if (kinds) {
        mixed_chunks(kinds, nq, chunk, &chunks, &maps);
    } else {
        for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
            MixedChunk c{};
            c.q0 = q0;
            c.q1 = std::min(nq, q0 + chunk);
            for (int j = 0; j < 3; ++j) {
                c.row0[j] = q0;
                c.rows[j] = p.use[j] ? c.q1 - q0 : 0;
            }
            chunks.push_back(c);
        }
    }
    uint32_t rmax[3] = {0, 0, 0};
    for (const MixedChunk &c : chunks)
        for (int j = 0; j < 3; ++j) rmax[j] = std::max(rmax[j], c.rows[j]);
    // per source: ids, scores, counts of a chunk's rows; then the maps and the dense error bytes
    const bool err_scratch = kinds && d_err && rmax[HYB_DENSE];
    size_t bytes = maps.size() * 4 + (err_scratch ? rmax[HYB_DENSE] : 0);
    for (int j = 0; j < 3; ++j) bytes += (size_t)rmax[j] * ((size_t)p.ld[j] * 8 + 4);
    const uint32_t dim = p.use[HYB_DENSE] ? index_dim(g->shard[0]) : 0;
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    const cudaStream_t s0 = slot_stream(g, 0, out_stream);
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s0));
    uint32_t *ids[3], *counts[3];
    float *scores[3];
    uint8_t *at = buf;
    for (int j = 0; j < 3; ++j) {
        ids[j] = reinterpret_cast<uint32_t *>(at);
        scores[j] = reinterpret_cast<float *>(ids[j] + (size_t)rmax[j] * p.ld[j]);
        counts[j] = reinterpret_cast<uint32_t *>(scores[j] + (size_t)rmax[j] * p.ld[j]);
        at = reinterpret_cast<uint8_t *>(counts[j] + rmax[j]);
    }
    uint32_t *d_maps = reinterpret_cast<uint32_t *>(at);
    uint8_t *err_dense = err_scratch ? reinterpret_cast<uint8_t *>(d_maps + maps.size()) : nullptr;
    cdb_status rc = CDB_OK;
    if (!maps.empty() && cudaMemcpyAsync(d_maps, maps.data(), maps.size() * 4, cudaMemcpyHostToDevice, s0) != cudaSuccess) {
        set_error("hybrid search: copying the row maps failed");
        rc = CDB_CUDA_ERROR;
    }
    const std::vector<ShardFilters> no_filters(nl, ShardFilters{nullptr, nullptr, 0, nullptr});
    std::vector<float *> idf;
    if (!rc && p.use[HYB_TFIDF]) rc = tfidf_idf_enqueue(g, tq, p.nq[HYB_TFIDF], nqh, &idf, out_stream);
    bool first = true;
    for (size_t ci = 0; ci < chunks.size() && !rc; ++ci) {
        const MixedChunk &c = chunks[ci];
        for (int j = 0; j < 3 && !rc; ++j) {
            const uint32_t r0 = c.row0[j], n = c.rows[j];
            if (!n) continue;
            // loopback: the slots write their gather buffers only after slot 0 copied the previous search's out of them
            if (!first && (rc = loopback_fence(g))) break;
            first = false;
            if (j == HYB_DENSE) {
                std::vector<const float *> q(nl);
                for (size_t i = 0; i < nl; ++i) q[i] = dq[i] + (size_t)r0 * dim;
                uint8_t *err = kinds ? err_dense : d_err ? d_err + c.q0 : nullptr;
                rc = sharded_enqueue(g, n, &p.dense, q, p.md ? &no_filters : nullptr, ids[j], scores[j], counts[j], err, out_stream);
            } else if (j == HYB_SPARSE) {
                std::vector<SparseQueries> q(nl);
                for (size_t i = 0; i < nl; ++i) q[i] = {sq[i].off + r0, sq[i].dims, sq[i].vals};
                rc = sparse_sharded_enqueue(g, n, &p.sparse, p.m, q, ids[j], scores[j], counts[j], out_stream);
            } else {
                rc = tfidf_sharded_enqueue(g, tq, nqh, idf, r0, n, k3, ids[j], scores[j], counts[j], out_stream);
            }
        }
        if (rc) break;
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        RrfList lists[3];
        for (int j = 0; j < 3; ++j) lists[j] = RrfList{ids[j], counts[j], p.ld[j], j == HYB_DENSE ? dense_id_stride : 1u};
        uint32_t *o_ids = d_ids + (size_t)c.q0 * ld_out, *o_counts = d_counts + c.q0;
        float *o_scores = d_scores + (size_t)c.q0 * ld_out;
        if (kinds) {
            rc = mixed_fuse(c, lists, d_maps, err_dense, fusion_k, ld_out, o_ids, o_scores, o_counts, d_err ? d_err + c.q0 : nullptr, s0);
        } else {
            const int f = p.use[HYB_DENSE] ? HYB_DENSE : HYB_SPARSE, s = p.use[HYB_TFIDF] ? HYB_TFIDF : HYB_SPARSE;
            const RrfList &a = lists[f], &b = lists[s];
            const uint32_t n = c.q1 - c.q0;
            if (!(rc = check_fuse_args(a.ld, b.ld, n, ld_out, a.ids, a.counts, b.ids, b.counts, o_ids, o_scores, o_counts)))
                rc = fuse_launch(a, b, n, fusion_k, ld_out, o_ids, o_scores, o_counts, s0);
        }
    }
    // freed behind everything enqueued on slot 0's stream, which every slot's last work joined (collective or loopback copy)
    tfidf_idf_free(g, idf, out_stream);
    cudaSetDevice(g->dev[0]);
    cudaFreeAsync(buf, s0);
    return rc;
}

cdb_status cdb_hybrid_search_batch_sharded(cdb_shard_group *g, const cdb_hybrid_group_sources *h, uint32_t nq, uint32_t top_k,
                                           float fusion_constant_k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts,
                                           uint8_t *err_flags) {
    CDB_REQUIRE(!nq || (out_counts && (!top_k || (out_ids && out_scores))), "null output");
    CDB_REQUIRE(g, "null group");
    HybPlan p;
    cdb_status rc = hyb_plan(h, nq, top_k, &p);
    if (rc || (rc = hyb_check_csr(h->sparse_offsets, h->sparse_dims, h->sparse_values, p.nq[HYB_SPARSE], h->tfidf_offsets,
                                  h->tfidf_hashes, p.nq[HYB_TFIDF])))
        return rc;
    std::lock_guard<std::mutex> lock(g->mu);
    if ((rc = hyb_group_check(g, &p))) return rc;
    if (!nq) return CDB_OK;
    if (!top_k) {
        memset(out_counts, 0, (size_t)nq * 4);
        return CDB_OK;
    }
    const size_t nl = g->dev.size();
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) {
        if (h->use_sparse) locks.emplace_back(sparse_index_mutex(g->sparse[i]));
        if (h->use_tfidf) locks.emplace_back(tfidf_index_mutex(g->tfidf[i]));
    }
    // the dense batch, the sparse CSR and the TF-IDF CSR of the named sources to every local device
    const uint32_t dim = h->use_dense ? index_dim(g->shard[0]) : 0;
    const uint64_t nqp = h->use_sparse ? h->sparse_offsets[nq] : 0, nqh = h->use_tfidf ? h->tfidf_offsets[nq] : 0;
    const size_t off_bytes = ((size_t)nq + 1) * 8;
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{h->dense_queries, (size_t)nq * dim * 4}, {h->sparse_offsets, h->use_sparse ? off_bytes : 0},
                                 {h->sparse_dims, nqp * 4}, {h->sparse_values, nqp * 4}, {h->tfidf_offsets, h->use_tfidf ? off_bytes : 0},
                                 {h->tfidf_hashes, nqh * 4}}, &st)) &&
        !(rc = host_rows(g, nq, 6 * top_k, out_ids, out_scores, out_counts, h->use_dense ? err_flags : nullptr, &r))) {
        std::vector<const float *> dq(nl);
        for (size_t i = 0; i < nl; ++i) dq[i] = st.at<float>(i, 0);
        rc = hybrid_group_run(g, p, nullptr, nq, top_k, fusion_constant_k, h->dense_id_stride, dq, staged_sparse(st, 1), staged_tfidf(st, 4),
                              nqh, r.ids, r.scores, r.counts, h->use_dense ? r.err : nullptr, nullptr);
    }
    return host_finish(g, rc, &r);
}

cdb_status cdb_hybrid_search_batch_sharded_device(cdb_shard_group *g, const cdb_hybrid_group_sources *h, uint32_t nq, uint32_t top_k,
                                                  float fusion_constant_k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                                  uint8_t *d_err_flags, void *stream) {
    CDB_REQUIRE(!nq || !top_k || (d_ids && d_scores && d_counts), "null output");
    CDB_REQUIRE(!nq || d_counts, "null output");
    CDB_REQUIRE(g, "null group");
    HybPlan p;
    cdb_status rc = hyb_plan(h, nq, top_k, &p);
    if (rc) return rc;
    if (h->use_tfidf) {
        set_error("the hybrid device form has no TF-IDF sub-search (the host sizes its idf exchange by the batch's term count, "
                  "which cdb_hybrid_group_sources does not carry): use cdb_hybrid_search_batch_sharded");
        return CDB_UNSUPPORTED;
    }
    CDB_REQUIRE(g->dev.size() == 1, "the device form serves groups of one local slot (cdb_shard_group_create_rank, or one device)");
    std::lock_guard<std::mutex> lock(g->mu);
    if ((rc = hyb_group_check(g, &p))) return rc;
    if (!nq) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    const cudaStream_t s = slot_stream(g, 0, (cudaStream_t)stream);
    if (!top_k) {
        CDB_CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, s));
        return CDB_OK;
    }
    std::unique_ptr<std::shared_lock<std::shared_mutex>> shard_lock;
    if (h->use_sparse) shard_lock.reset(new std::shared_lock<std::shared_mutex>(sparse_index_mutex(g->sparse[0])));
    const std::vector<const float *> dq(1, h->dense_queries);
    const std::vector<SparseQueries> sq(1, SparseQueries{h->sparse_offsets, h->sparse_dims, h->sparse_values});
    return hybrid_group_run(g, p, nullptr, nq, top_k, fusion_constant_k, h->dense_id_stride, dq, sq, {}, 0, d_ids, d_scores, d_counts,
                            h->use_dense ? d_err_flags : nullptr, (cudaStream_t)stream);
}

cdb_status cdb_hybrid_search_batch_mixed_sharded(cdb_shard_group *g, const cdb_hybrid_group_mixed_sources *h, uint32_t nq, uint32_t top_k,
                                                 float fusion_constant_k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts,
                                                 uint8_t *err_flags) {
    CDB_REQUIRE(!nq || (out_counts && (!top_k || (out_ids && out_scores))), "null output");
    CDB_REQUIRE(g, "null group");
    HybPlan p;
    cdb_status rc = hyb_mixed_plan(h, nq, top_k, &p);
    if (rc || (rc = hyb_check_csr(h->sparse_offsets, h->sparse_dims, h->sparse_values, h->n_sparse, h->tfidf_offsets, h->tfidf_hashes,
                                  h->n_tfidf)))
        return rc;
    std::lock_guard<std::mutex> lock(g->mu);
    if ((rc = hyb_group_check(g, &p))) return rc;
    if (!nq) return CDB_OK;
    if (!top_k) {
        memset(out_counts, 0, (size_t)nq * 4);
        return CDB_OK;
    }
    const size_t nl = g->dev.size();
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    for (size_t i = 0; i < nl; ++i) {
        if (p.use[HYB_SPARSE]) locks.emplace_back(sparse_index_mutex(g->sparse[i]));
        if (p.use[HYB_TFIDF]) locks.emplace_back(tfidf_index_mutex(g->tfidf[i]));
    }
    // each source's batch to every local device, once
    const uint32_t dim = p.use[HYB_DENSE] ? index_dim(g->shard[0]) : 0;
    const uint64_t nqp = h->n_sparse ? h->sparse_offsets[h->n_sparse] : 0, nqh = h->n_tfidf ? h->tfidf_offsets[h->n_tfidf] : 0;
    Staged st;
    HostRows r;
    if (!(rc = stage_queries(g, {{h->dense_queries, (size_t)h->n_dense * dim * 4},
                                 {h->sparse_offsets, h->n_sparse ? ((size_t)h->n_sparse + 1) * 8 : 0}, {h->sparse_dims, nqp * 4},
                                 {h->sparse_values, nqp * 4}, {h->tfidf_offsets, h->n_tfidf ? ((size_t)h->n_tfidf + 1) * 8 : 0},
                                 {h->tfidf_hashes, nqh * 4}}, &st)) &&
        !(rc = host_rows(g, nq, 6 * top_k, out_ids, out_scores, out_counts, err_flags, &r))) {
        std::vector<const float *> dq(nl);
        for (size_t i = 0; i < nl; ++i) dq[i] = st.at<float>(i, 0);
        rc = hybrid_group_run(g, p, h->kinds, nq, top_k, fusion_constant_k, h->dense_id_stride, dq, staged_sparse(st, 1), staged_tfidf(st, 4),
                              nqh, r.ids, r.scores, r.counts, err_flags ? r.err : nullptr, nullptr);
    }
    return host_finish(g, rc, &r);
}

cdb_status cdb_hybrid_search_batch_mixed_sharded_device(cdb_shard_group *g, const cdb_hybrid_group_mixed_sources *h, uint32_t nq,
                                                        uint32_t top_k, float fusion_constant_k, uint32_t *d_ids, float *d_scores,
                                                        uint32_t *d_counts, uint8_t *d_err_flags, void *stream) {
    CDB_REQUIRE(!nq || (d_counts && (!top_k || (d_ids && d_scores))), "null output");
    CDB_REQUIRE(g, "null group");
    HybPlan p;
    cdb_status rc = hyb_mixed_plan(h, nq, top_k, &p);
    if (rc) return rc;
    CDB_REQUIRE(!h->n_tfidf || h->tfidf_hashes || !h->n_tfidf_hashes, "null tf-idf query hashes");
    CDB_REQUIRE(h->n_tfidf_hashes < (1ull << 31), "a batch of 2^31 query terms or more");
    CDB_REQUIRE(g->dev.size() == 1, "the device form serves groups of one local slot (cdb_shard_group_create_rank, or one device)");
    std::lock_guard<std::mutex> lock(g->mu);
    if ((rc = hyb_group_check(g, &p))) return rc;
    if (!nq) return CDB_OK;
    // the group's work follows what the caller's stream held, and the caller's later work follows it
    const cudaStream_t out = (cudaStream_t)stream, s = slot_stream(g, 0, out);
    CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
    if (s != out) {
        CDB_CUDA_TRY(cudaEventRecord(g->ev[0], out));
        CDB_CUDA_TRY(cudaStreamWaitEvent(s, g->ev[0], 0));
    }
    if (!top_k) {
        rc = cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, s) == cudaSuccess ? CDB_OK : CDB_CUDA_ERROR;
        if (rc) set_error("hybrid search: cudaMemsetAsync failed");
    } else {
        std::vector<std::shared_lock<std::shared_mutex>> locks;
        if (p.use[HYB_SPARSE]) locks.emplace_back(sparse_index_mutex(g->sparse[0]));
        if (p.use[HYB_TFIDF]) locks.emplace_back(tfidf_index_mutex(g->tfidf[0]));
        rc = hybrid_group_run(g, p, h->kinds, nq, top_k, fusion_constant_k, h->dense_id_stride, {h->dense_queries},
                              {SparseQueries{h->sparse_offsets, h->sparse_dims, h->sparse_values}},
                              {TfQueries{h->tfidf_offsets, h->tfidf_hashes}}, h->n_tfidf_hashes, d_ids, d_scores, d_counts, d_err_flags, out);
    }
    if (s != out) {
        CDB_CUDA_TRY(cudaSetDevice(g->dev[0]));
        CDB_CUDA_TRY(cudaEventRecord(g->ev[0], s));
        CDB_CUDA_TRY(cudaStreamWaitEvent(out, g->ev[0], 0));
    }
    return rc;
}

}  // extern "C"
