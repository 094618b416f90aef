// tfidf.cu -- the TF-IDF / BM25 index (TFIDFIndex, src/indexes/tf_idf/mod.rs) on the GPU: ingest and versioned deletes of
// (term_hash, tf) documents (TFIDFIndexRoot::insert / delete, src/models/tf_idf_index.rs:315-352, on the VersionedVec of
// src/models/versioned_vec.rs) and SparseAnnQueryBasic::search_bm25 (src/models/sparse_ann_query.rs:149-233) with get_idf
// (sparse_ann_query.rs:298-302).  The contract is the header comment of cdb_tfidf_index_create.
//
// Layout (DESIGN.md section 8d).  The rows and posting tiles are a PostingTiles store (posting_tiles.cuh) keyed by term
// hash, with entries (row_in_tile, tf bits), ascending by row inside a segment.  The host keeps the sorted table of every
// hash the index has seen with its df (VersionedVec::len) and uploads the table and its df after every append and delete;
// a kernel then computes the idf of every term on the device (bm25_idf.h).  A search scores one (query, tile) per CTA into
// shared-memory f32 accumulators plus a touched flag per row, query terms strictly in the caller's order, reduces the tile
// to its 512 bucket winners, then merges the tiles per bucket and sorts the winners.
#include <algorithm>
#include <cmath>
#include <mutex>
#include <shared_mutex>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

#include "bm25_idf.h"
#include "kernels.h"
#include "posting_tiles.cuh"
#include "tfidf_file.h"

namespace cdb {
namespace {

constexpr int TF_THREADS = 512;
constexpr uint32_t TF_BUCKETS = 512;       // search_bm25's BUCKETS
constexpr uint32_t TF_QCHUNK = TF_THREADS; // query terms resolved per pass of the scoring kernel
static_assert(TF_THREADS == (int)TF_BUCKETS, "one thread per bucket in the tile reduction and the final sort");

// posting entries (row_in_tile, tf bits), sorted on hash << 15 | row: ascending rows inside a hash's segment.  Equal sort
// keys are a row that repeats a hash.
struct TfCodec {
    using Entry = uint2;
    static constexpr int END_BIT = 32 + TILE_SHIFT, SEG_SHIFT = TILE_SHIFT;
    static constexpr const char *DUPLICATE_ERROR = "a row repeats a term hash";
    __device__ SortPair encode(uint32_t hash, float tf, uint32_t row) const {
        return {((uint64_t)hash << TILE_SHIFT) | row, __float_as_uint(tf)};
    }
    __device__ Entry entry(uint64_t k, uint32_t v) const { return make_uint2((uint32_t)(k & (TILE_ROWS - 1)), v); }
};

// the hashes of rows[0..n) packed at out[off[i] ..] (one warp per row)
__global__ void tf_gather_rows_kernel(const uint64_t *__restrict__ row_off, const uint32_t *__restrict__ hashes,
                                      const uint32_t *__restrict__ rows, const uint64_t *__restrict__ off, uint32_t n,
                                      uint32_t *__restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n) return;
    const uint64_t b = row_off[rows[warp]], e = row_off[rows[warp] + 1];
    for (uint64_t p = b + lane; p < e; p += 32) out[off[warp] + (p - b)] = hashes[p];
}

// ---------------------------------------------------------------- search side
struct TfSearch {
    const uint2 *entries;
    const uint32_t *thash, *tseg, *deleted;
    const PostingTile *tiles;
    const uint32_t *terms;   // every hash the index has seen, ascending
    const float *idf;        // idf of terms[i]
    const float *q_idf;      // NULL, or the idf of every query term (a shard group's global idf), used for terms this index holds
    uint32_t n_terms;
    uint64_t n_rows;
    uint32_t id_base;
    const uint64_t *q_off;
    const uint32_t *q_hash;
    uint64_t q_end;          // query terms the caller's arrays hold: no term at or past it is read, whatever q_off says
    uint32_t q0;             // first query of the chunk
    uint32_t n_tiles;
    uint2 *out;              // [chunk][n_tiles][512] bucket winners (id, score bits); id CDB_INVALID_ID = empty
};

constexpr size_t TF_SCORE_SMEM = (size_t)TILE_ROWS * 4 + TILE_ROWS + (size_t)TF_QCHUNK * 12;

__global__ void __launch_bounds__(TF_THREADS, 1) tf_score_tile_kernel(TfSearch a) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *acc = reinterpret_cast<float *>(smem);
    uint8_t *touched = smem + (size_t)TILE_ROWS * 4;
    uint32_t *c_beg = reinterpret_cast<uint32_t *>(touched + TILE_ROWS);   // segment of each resolved term (tile-relative)
    uint32_t *c_len = c_beg + TF_QCHUNK;
    float *c_idf = reinterpret_cast<float *>(c_len + TF_QCHUNK);

    const uint32_t t = blockIdx.x, qi = blockIdx.y, q = a.q0 + qi, tid = threadIdx.x;
    const PostingTile tile = a.tiles[t];
    const uint64_t row0 = (uint64_t)t << TILE_SHIFT;
    const uint32_t nr = (uint32_t)std::min<uint64_t>(TILE_ROWS, a.n_rows - row0);
    uint4 *t4 = reinterpret_cast<uint4 *>(touched);
    for (uint32_t i = tid; i < TILE_ROWS / 16; i += TF_THREADS) t4[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();

    const uint32_t *thash = a.thash + tile.key_base;
    const uint32_t *tseg = a.tseg + tile.key_base + t;
    const uint2 *ent = a.entries + tile.entry_base;
    const uint64_t qe = min(a.q_off[q + 1], a.q_end), qb = min(a.q_off[q], qe);
    for (uint64_t j0 = qb; j0 < qe; j0 += TF_QCHUNK) {
        const uint32_t nj = (uint32_t)std::min<uint64_t>(TF_QCHUNK, qe - j0);
        if (tid < nj) {
            // search_bm25's head for this term: absent terms are skipped, a present one carries get_idf of its list
            const uint32_t h = a.q_hash[j0 + tid];
            const uint32_t g = lower_bound_u32(a.terms, a.n_terms, h);
            uint32_t s = 0, e = 0;
            float idf = 0.0f;
            if (g < a.n_terms && a.terms[g] == h) {
                idf = a.q_idf ? a.q_idf[j0 + tid] : a.idf[g];
                const uint32_t l = lower_bound_u32(thash, tile.n_keys, h);
                if (l < tile.n_keys && thash[l] == h) { s = tseg[l]; e = tseg[l + 1]; }
            }
            c_beg[tid] = s;
            c_len[tid] = e - s;
            c_idf[tid] = idf;
        }
        __syncthreads();
        // the terms in the caller's order; inside one segment every row appears once, so each thread owns its rows
        for (uint32_t j = 0; j < nj; ++j) {
            const uint32_t beg = c_beg[j], len = c_len[j];
            const float idf = c_idf[j];
            for (uint32_t i = tid; i < len; i += TF_THREADS) {
                const uint2 e = __ldg(ent + beg + i);
                const float p = __fmul_rn(__uint_as_float(e.y), idf);
                if (touched[e.x]) {
                    acc[e.x] = __fadd_rn(acc[e.x], p);
                } else {
                    acc[e.x] = p;   // the first product, not 0 + product: a -0 score keeps its sign
                    touched[e.x] = 1;
                }
            }
            __syncthreads();
        }
    }
    // bucket id % 512: the rows of one bucket, visited in ascending id; `score > best` from -inf keeps the first of equal
    // scores and never admits NaN or -inf.  Deleted rows are skipped.
    const uint32_t id0 = a.id_base + (uint32_t)row0;
    float best = -INFINITY;
    uint32_t bid = CDB_INVALID_ID;
    for (uint32_t r = (tid - id0) & (TF_BUCKETS - 1); r < nr; r += TF_BUCKETS) {
        if (!touched[r]) continue;
        const uint64_t g = row0 + r;
        if (a.deleted && (a.deleted[g >> 5] >> (g & 31)) & 1u) continue;
        const float s = acc[r];
        if (s > best) { best = s; bid = id0 + r; }
    }
    a.out[((size_t)qi * a.n_tiles + t) * TF_BUCKETS + tid] = make_uint2(bid, __float_as_uint(best));
}

// bucket threadIdx.x's winner over the tiles of one query (src = its [n_tiles][512] winners), merged in ascending tile
// order: ascending ids, so `>` keeps the reference's winner.  (CDB_INVALID_ID, -inf) when the bucket is empty.
__device__ __forceinline__ uint2 tf_bucket_winner(const uint2 *__restrict__ src, uint32_t n_tiles) {
    float best = -INFINITY;
    uint32_t bid = CDB_INVALID_ID;
    for (uint32_t t = 0; t < n_tiles; ++t) {
        const uint2 w = src[(size_t)t * TF_BUCKETS + threadIdx.x];
        const float s = __uint_as_float(w.y);
        if (w.x != CDB_INVALID_ID && s > best) { best = s; bid = w.x; }
    }
    return make_uint2(bid, __float_as_uint(best));
}

// idf[i] = bm25_idf(n_docs, df[i]): the index's idf table after an append or a delete
__global__ void tf_idf_table_kernel(const uint32_t *__restrict__ df, uint32_t n, uint32_t n_docs, float *__restrict__ idf) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idf[i] = bm25_idf(n_docs, df[i]);
}

// one shard's statistics for a shard group's idf: out = [n_docs, df of hashes[0..n)] (u32; 0 for a hash the shard never saw)
__global__ void tf_query_stats_kernel(const uint32_t *__restrict__ terms, const uint32_t *__restrict__ df, uint32_t n_terms,
                                      uint32_t n_docs, const uint32_t *__restrict__ hashes, uint64_t n, uint32_t *__restrict__ out) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) out[0] = n_docs;
    if (j >= n) return;
    const uint32_t h = hashes[j];
    const uint32_t g = lower_bound_u32(terms, n_terms, h);
    out[1 + j] = g < n_terms && terms[g] == h ? df[g] : 0u;
}

// a shard group's idf of every query term: N and df summed over the ranks' statistics (rank r's at gathered + r * words,
// u32, wrapping), then bm25_idf
__global__ void tf_group_idf_kernel(const uint64_t *__restrict__ gathered, size_t words, uint32_t world, uint64_t n,
                                    float *__restrict__ q_idf) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint32_t n_docs = 0, df = 0;
    for (uint32_t r = 0; r < world; ++r) {
        const uint32_t *st = reinterpret_cast<const uint32_t *>(gathered + r * words);
        n_docs += st[0];
        df += st[1 + j];
    }
    q_idf[j] = bm25_idf(n_docs, df);
}

// cdb_debug_bm25's device form: the bm25_log1pf and bm25_idf the two kernels above inline, over arrays (grid-stride)
__global__ void tf_debug_bm25_kernel(const float *__restrict__ x, uint64_t n, float *__restrict__ out_log1p,
                                     const uint32_t *__restrict__ n_docs, const uint32_t *__restrict__ df, uint64_t n_pairs,
                                     float *__restrict__ out_idf) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out_log1p[i] = bm25_log1pf(x[i]);
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_pairs; j += stride) out_idf[j] = bm25_idf(n_docs[j], df[j]);
}

// one shard's half of a shard group's search: every bucket's winner per query, [nq][512], neither sorted nor truncated
__global__ void __launch_bounds__(TF_THREADS, 1) tf_winners_kernel(const uint2 *__restrict__ in, uint32_t n_tiles, uint2 *__restrict__ out) {
    out[(size_t)blockIdx.x * TF_BUCKETS + threadIdx.x] = tf_bucket_winner(in + (size_t)blockIdx.x * n_tiles * TF_BUCKETS, n_tiles);
}

// the <= 512 bucket winners of one query (thread = bucket) sorted by total_cmp descending, ties to the smaller id, truncated
// to kout and written out
__device__ __forceinline__ void tf_sort_winners(uint2 win, uint32_t kout, uint32_t *__restrict__ out_ids, float *__restrict__ out_scores,
                                                uint32_t *__restrict__ out_count) {
    __shared__ uint64_t keys[TF_BUCKETS];
    __shared__ uint32_t s_cnt;
    const uint32_t tid = threadIdx.x, bid = win.x;
    const float best = __uint_as_float(win.y);
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    // order_key of a non-NaN score is non-zero above -inf's; 0 marks an empty bucket
    keys[tid] = bid == CDB_INVALID_ID ? 0ull
                                      : ((uint64_t)order_key(CDB_METRIC_DOT_PRODUCT, __float_as_uint(best)) << 32) | (uint64_t)(~bid);
    if (bid != CDB_INVALID_ID) atomicAdd(&s_cnt, 1u);
    __syncthreads();
    bitonic_sort<true>(keys, TF_BUCKETS);
    const uint32_t cnt = min(s_cnt, kout);
    if (tid < kout) {
        uint32_t id = CDB_INVALID_ID;
        float s = 0.0f;
        if (tid < cnt) {
            const uint64_t key = keys[tid];
            id = ~(uint32_t)key;
            s = __uint_as_float(key_to_bits(CDB_METRIC_DOT_PRODUCT, (uint32_t)(key >> 32)));
        }
        out_ids[tid] = id;
        out_scores[tid] = s;
    }
    if (tid == 0) *out_count = cnt;
}

// per query: the tiles' winners of each bucket, then sorted and truncated to kout
__global__ void __launch_bounds__(TF_THREADS, 1) tf_finalize_kernel(const uint2 *__restrict__ in, uint32_t n_tiles, uint32_t kout,
                                                                     uint32_t *__restrict__ out_ids, float *__restrict__ out_scores,
                                                                     uint32_t *__restrict__ out_counts) {
    const uint32_t qi = blockIdx.x;
    tf_sort_winners(tf_bucket_winner(in + (size_t)qi * n_tiles * TF_BUCKETS, n_tiles), kout, out_ids + (size_t)qi * kout,
                    out_scores + (size_t)qi * kout, out_counts + qi);
}

// a shard group's merge: per query and bucket the best of the ranks' winners (gathered, rank r's [nq][512] at r * words),
// `score > best` with equal scores (+0 and -0 too) going to the smaller id, since rank order need not follow id order;
// then sorted and truncated as tf_finalize_kernel does
__global__ void __launch_bounds__(TF_THREADS, 1) tf_group_finalize_kernel(const uint2 *__restrict__ gathered, size_t words, uint32_t world,
                                                                           uint32_t kout, uint32_t *__restrict__ out_ids,
                                                                           float *__restrict__ out_scores, uint32_t *__restrict__ out_counts) {
    const uint32_t qi = blockIdx.x;
    float best = -INFINITY;
    uint32_t bid = CDB_INVALID_ID;
    for (uint32_t r = 0; r < world; ++r) {
        const uint2 w = gathered[r * words + (size_t)qi * TF_BUCKETS + threadIdx.x];
        const float s = __uint_as_float(w.y);
        if (w.x != CDB_INVALID_ID && (s > best || (s == best && w.x < bid))) { best = s; bid = w.x; }
    }
    tf_sort_winners(make_uint2(bid, __float_as_uint(best)), kout, out_ids + (size_t)qi * kout, out_scores + (size_t)qi * kout, out_counts + qi);
}

// ---------------------------------------------------------------- load from the reference's files (cdb_tfidf_index_load_files)
// One staged chunk of the files' record words, positions pos0 .. pos0 + n of their concatenation (marked words already
// u64::MAX): every live word whose id is in [id_base, id_base + n_rows), as the sort key row << 32 | hash and the value
// version << 32 | tf bits, compacted at *count with one atomic per warp (the order is settled by the sort that follows, whose
// keys are unique unless a row repeats a hash).  Nothing is written at or past cap.  rec_base / rec_meta: each record's
// first position and (hash, version), ascending positions.
__global__ void tf_load_decode_kernel(const uint64_t *__restrict__ words, uint64_t n, uint64_t pos0, const uint64_t *__restrict__ rec_base,
                                      const uint2 *__restrict__ rec_meta, uint32_t n_recs, uint32_t id_base, uint64_t n_rows, uint64_t cap,
                                      unsigned long long *__restrict__ count, uint64_t *__restrict__ keys, uint64_t *__restrict__ vals) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint64_t w = ~0ull, row = 0;
        bool take = false;
        if (i < n) {
            w = words[i];
            row = (uint64_t)(uint32_t)(w >> 32) - id_base;   // wraps past n_rows below id_base
            take = w != ~0ull && !(w >> 63) && row < n_rows;
        }
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, take);
        if (!m) continue;
        const int leader = __ffs(m) - 1;
        unsigned long long at = 0;
        if (lane == (uint32_t)leader) at = atomicAdd(count, (unsigned long long)__popc(m));
        at = __shfl_sync(0xFFFFFFFFu, at, leader) + __popc(m & ((1u << lane) - 1));
        if (!take || at >= cap) continue;
        // the record holding position pos0 + i: the last one starting at or before it
        const uint64_t pos = pos0 + i;
        uint32_t lo = 0, hi = n_recs;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (rec_base[mid] <= pos) lo = mid + 1; else hi = mid; }
        const uint2 meta = rec_meta[lo - 1];
        keys[at] = row << 32 | meta.x;
        vals[at] = (uint64_t)meta.y << 32 | (uint32_t)w;
    }
}

// row_off[r], r in [0, n_rows]: the first of the n sorted keys whose row is r or more
__global__ void tf_load_offsets_kernel(const uint64_t *__restrict__ keys, uint64_t n, uint64_t n_rows, uint64_t *__restrict__ row_off) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    uint64_t lo = 0, hi = n;
    while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if ((keys[mid] >> 32) < r) lo = mid + 1; else hi = mid; }
    row_off[r] = lo;
}

// the sorted pairs into the store's hashes and tf values, the version of each row's first pair into row_version, and
// *mixed = 1 when a row's pairs carry two versions
__global__ void tf_load_rows_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ vals, uint64_t n,
                                    uint32_t *__restrict__ out_hashes, float *__restrict__ out_tfs, uint32_t *__restrict__ row_version,
                                    uint32_t *__restrict__ mixed) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = keys[i], v = vals[i];
    out_hashes[i] = (uint32_t)k;
    out_tfs[i] = __uint_as_float((uint32_t)v);
    if (i == 0 || (keys[i - 1] >> 32) != (k >> 32)) row_version[k >> 32] = (uint32_t)(v >> 32);
    else if ((vals[i - 1] >> 32) != (v >> 32)) *mixed = 1u;
}

}  // namespace
}  // namespace cdb

using namespace cdb;

struct cdb_tfidf_index {
    cdb_tfidf_index_desc desc;
    std::shared_mutex rw;
    PostingTiles<TfCodec> st;        // keys: term hashes
    uint32_t documents = 0;          // total_documents_count
    uint32_t version = 0;            // the latest version passed to append / delete_rows
    std::vector<uint8_t> h_counted;
    std::vector<uint32_t> h_version; // insert version per row
    std::vector<uint32_t> h_terms;   // every hash seen, ascending
    std::vector<uint32_t> h_df;      // VersionedVec::len of each
    uint32_t *d_terms = nullptr;
    uint32_t *d_df = nullptr;        // h_df on the device
    float *d_idf = nullptr;          // bm25_idf(documents, d_df[i])
    uint64_t terms_cap = 0;
    ~cdb_tfidf_index() {
        if (d_terms) cudaFree(d_terms);
        if (d_df) cudaFree(d_df);
        if (d_idf) cudaFree(d_idf);
    }
};

namespace {

// the term table and its df to the device, and the idf under `n_docs` computed there (the device is idle: the caller holds
// the handle exclusively and has drained queued searches)
cdb_status upload_terms(cdb_tfidf_index *ix, const std::vector<uint32_t> &terms, const std::vector<uint32_t> &df, uint32_t n_docs,
                        bool terms_changed, cudaStream_t s) {
    const size_t n = terms.size();
    if (n > ix->terms_cap) {
        const uint64_t cap = std::max<uint64_t>(n, 2 * ix->terms_cap);
        uint32_t *t = nullptr, *d = nullptr;
        float *f = nullptr;
        CDB_CUDA_TRY(cudaMalloc(&t, cap * 4));
        cudaError_t e = cudaMalloc(&d, cap * 4);
        if (e == cudaSuccess) e = cudaMalloc(&f, cap * 4);
        if (e != cudaSuccess) {
            cudaFree(t);
            if (d) cudaFree(d);
            set_error(std::string("cudaMalloc: ") + cudaGetErrorString(e));
            return CDB_CUDA_ERROR;
        }
        if (ix->d_terms) cudaFree(ix->d_terms);
        if (ix->d_df) cudaFree(ix->d_df);
        if (ix->d_idf) cudaFree(ix->d_idf);
        ix->d_terms = t;
        ix->d_df = d;
        ix->d_idf = f;
        ix->terms_cap = cap;
        terms_changed = true;
    }
    if (!n) return CDB_OK;
    if (terms_changed) CDB_CUDA_TRY(cudaMemcpyAsync(ix->d_terms, terms.data(), n * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(ix->d_df, df.data(), n * 4, cudaMemcpyHostToDevice, s));
    tf_idf_table_kernel<<<(uint32_t)((n + 255) / 256), 256, 0, s>>>(ix->d_df, (uint32_t)n, n_docs, ix->d_idf);
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

// the distinct hashes of d_hashes[0..np) ascending into uniq, and how many pairs hold each into cnt, then a drain of s.  b's
// scratch must hold np pairs: sorted hashes -> b.vals_out, distinct -> b.flags, counts -> b.vals_in, their number -> b.pos
cudaError_t distinct_hashes(const uint32_t *d_hashes, uint64_t np, BuildBufs &b, cudaStream_t s, std::vector<uint32_t> &uniq,
                            std::vector<uint32_t> &cnt) {
    cudaError_t e = cudaSuccess;
    if (np) {
        uint32_t *runs = b.pos;
        size_t t_sort = 0, t_rle = 0;
        e = cub::DeviceRadixSort::SortKeys(nullptr, t_sort, d_hashes, b.vals_out, (int)np, 0, 32, s);
        if (e == cudaSuccess) e = cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, b.vals_out, b.flags, b.vals_in, runs, (int)np, s);
        const size_t need = std::max(t_sort, t_rle);
        void *tmp = b.tmp;
        if (e == cudaSuccess && need > b.tmp_bytes) e = cudaMallocAsync(&tmp, need, s);
        size_t tb = need;
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortKeys(tmp, tb, d_hashes, b.vals_out, (int)np, 0, 32, s);
        tb = need;
        if (e == cudaSuccess) e = cub::DeviceRunLengthEncode::Encode(tmp, tb, b.vals_out, b.flags, b.vals_in, runs, (int)np, s);
        uint32_t n_runs = 0;
        if (e == cudaSuccess) e = cudaMemcpyAsync(&n_runs, runs, 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess) {
            uniq.resize(n_runs);
            cnt.resize(n_runs);
            e = cudaMemcpyAsync(uniq.data(), b.flags, n_runs * 4ull, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(cnt.data(), b.vals_in, n_runs * 4ull, cudaMemcpyDeviceToHost, s);
        }
        if (tmp != b.tmp) cudaFreeAsync(tmp, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return e;
}

uint32_t out_cols(uint32_t k) { return (k == 0 || k > TF_BUCKETS) ? TF_BUCKETS : k; }

// the scoring kernel's arguments for queries [q0, q0 + chunk); q_idf as TfSearch::q_idf
TfSearch score_args(const cdb_tfidf_index *ix, const uint64_t *d_qoff, const uint32_t *d_qhash, uint64_t q_end, const float *q_idf, uint32_t q0,
                    uint2 *win) {
    TfSearch a;
    a.entries = ix->st.entries(); a.thash = ix->st.d_tkeys; a.tseg = ix->st.d_tseg; a.deleted = ix->st.deleted();
    a.tiles = ix->st.d_tiles; a.terms = ix->d_terms; a.idf = ix->d_idf; a.q_idf = q_idf; a.n_terms = (uint32_t)ix->h_terms.size();
    a.n_rows = ix->st.n_rows; a.id_base = ix->desc.id_base; a.q_off = d_qoff; a.q_hash = d_qhash; a.q_end = q_end; a.q0 = q0;
    a.n_tiles = (uint32_t)ix->st.h_tiles.size(); a.out = win;
    return a;
}

// queries per chunk and the tile winners' scratch of one chunk
uint32_t score_chunk(uint32_t nq, uint32_t n_tiles, size_t *per_q) {
    *per_q = (size_t)n_tiles * TF_BUCKETS * sizeof(uint2);
    return (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)nq, 65535, (512ull << 20) / *per_q}));
}

cdb_status search_locked(cdb_tfidf_index *ix, const uint64_t *d_qoff, const uint32_t *d_qhash, uint32_t nq, uint32_t k,
                         uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t s) {
    if (!nq) return CDB_OK;
    const uint32_t kout = out_cols(k);
    const uint32_t n_tiles = (uint32_t)ix->st.h_tiles.size();
    if (n_tiles == 0) return fill_empty_results(nq, kout, d_ids, d_scores, d_counts, s);
    size_t per_q = 0;
    const uint32_t chunk = score_chunk(nq, n_tiles, &per_q);
    uint2 *win = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&win, (size_t)chunk * per_q, s));
    cdb_status rc = CDB_OK;
    cudaError_t e = allow_max_dynamic_smem((const void *)tf_score_tile_kernel);
    if (e != cudaSuccess) { set_error(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    for (uint32_t q0 = 0; q0 < nq && !rc; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        tf_score_tile_kernel<<<dim3(n_tiles, c), TF_THREADS, TF_SCORE_SMEM, s>>>(score_args(ix, d_qoff, d_qhash, UINT64_MAX, nullptr, q0, win));
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; break; }
        tf_finalize_kernel<<<c, TF_THREADS, 0, s>>>(win, n_tiles, kout, d_ids + (size_t)q0 * kout, d_scores + (size_t)q0 * kout,
                                                     d_counts + q0);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(win, s);
    return rc;
}

constexpr uint64_t TF_LOAD_STAGE_WORDS = (128ull << 20) / 8;   // two pinned staging buffers of 128 MB each

// cdb_tfidf_index_load_files past its checks, on an empty index held exclusively, with the device drained.  The caller
// empties the store again if this fails.
cdb_status load_locked(cdb_tfidf_index *ix, const cdb_tfidf_files *f, uint64_t n_rows, const uint8_t *counted, bool carry, cudaStream_t s) {
    PostingTiles<TfCodec> &st = ix->st;
    const uint64_t n_recs = f->recs.size(), n_words = f->n_words;
    CDB_REQUIRE(n_recs < (1ull << 32), "tf-idf load: the files hold 2^32 list records or more");
    const uint64_t cap = std::min<uint64_t>(f->n_live, st.capacity_pairs);
    const uint64_t stage = std::min<uint64_t>(n_words, TF_LOAD_STAGE_WORDS);
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ix->desc.device));
    // device scratch: record table, two sort buffers of cap keys and values, staging, the count, the row versions, the flag
    const size_t bytes = n_recs * 16 + cap * 32 + 2 * stage * 8 + 8 + n_rows * 4 + 4;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    uint64_t *rec_base = reinterpret_cast<uint64_t *>(buf);
    uint2 *rec_meta = reinterpret_cast<uint2 *>(rec_base + n_recs);
    uint64_t *k0 = reinterpret_cast<uint64_t *>(rec_meta + n_recs), *k1 = k0 + cap, *v0 = k1 + cap, *v1 = v0 + cap;
    uint64_t *d_stage = v1 + cap;
    unsigned long long *d_count = reinterpret_cast<unsigned long long *>(d_stage + 2 * stage);
    uint32_t *row_version = reinterpret_cast<uint32_t *>(d_count + 1);
    uint32_t *d_mixed = row_version + n_rows;
    uint64_t *h_stage = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    void *tmp = nullptr;
    auto done = [&](cudaError_t e) -> cdb_status {
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (tmp) cudaFreeAsync(tmp, s);
        cudaFreeAsync(buf, s);
        cudaStreamSynchronize(s);
        if (h_stage) cudaFreeHost(h_stage);
        for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x);
        if (e != cudaSuccess) { set_error(std::string("tf-idf load: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
        return CDB_OK;
    };
    // the record table, then the words in chunks: copied into pinned memory record by record, the marked words overwritten
    // with u64::MAX, uploaded and decoded while the host fills the other buffer
    std::vector<uint64_t> hb(n_recs);
    std::vector<uint2> hm(n_recs);
    for (uint64_t r = 0; r < n_recs; ++r) { hb[r] = f->recs[r].base; hm[r] = make_uint2(f->hashes[f->recs[r].term], f->recs[r].version); }
    cudaError_t e = cudaMemsetAsync(d_count, 0, 8, s);
    if (e == cudaSuccess && n_recs) e = cudaMemcpyAsync(rec_base, hb.data(), n_recs * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_recs) e = cudaMemcpyAsync(rec_meta, hm.data(), n_recs * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && stage) e = cudaHostAlloc(&h_stage, 2 * stage * 8, cudaHostAllocDefault);
    for (int i = 0; i < 2 && e == cudaSuccess && stage; ++i) e = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming);
    uint64_t ri = 0, within = 0;
    size_t k = 0;
    for (uint64_t c0 = 0, it = 0; c0 < n_words && e == cudaSuccess; c0 += stage, ++it) {
        const uint64_t nw = std::min(stage, n_words - c0);
        const int half = (int)(it & 1);
        uint64_t *h = h_stage + half * stage;
        if (it >= 2 && (e = cudaEventSynchronize(ev[half])) != cudaSuccess) break;
        for (uint64_t filled = 0; filled < nw;) {
            const TfIdfFileRecord &r = f->recs[ri];
            const uint64_t take = std::min<uint64_t>(r.len - within, nw - filled);
            memcpy(h + filled, r.words + 8 * within, take * 8);
            filled += take;
            within += take;
            if (within == r.len) { ++ri; within = 0; }
        }
        for (; k < f->killed.size() && f->killed[k] < c0 + nw; ++k) h[f->killed[k] - c0] = ~0ull;
        e = cudaMemcpyAsync(d_stage + half * stage, h, nw * 8, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaEventRecord(ev[half], s);
        if (e != cudaSuccess) break;
        const uint32_t blocks = (uint32_t)std::min<uint64_t>((nw + 255) / 256, (uint64_t)sms * 16);   // grid-stride
        tf_load_decode_kernel<<<blocks, 256, 0, s>>>(d_stage + half * stage, nw, c0, rec_base, rec_meta, (uint32_t)n_recs, ix->desc.id_base,
                                                      n_rows, cap, d_count, k0, v0);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    unsigned long long np = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&np, d_count, 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return done(e);
    if (np > st.capacity_pairs || np >= (1ull << 31)) {
        done(cudaSuccess);
        set_error("tf-idf load: the files hold " + std::to_string(np) + " live pairs for these rows, more than capacity_pairs or 2^31 - 1");
        return CDB_INVALID_PARAMS;
    }
    // rows: the pairs sorted on row << 32 | hash (each row ascending by hash), the offsets, the store's pairs, the versions
    const int end_bit = 32 + (n_rows > 1 ? 64 - __builtin_clzll(n_rows - 1) : 0);
    if (np) {
        size_t tb = 0;
        e = cub::DeviceRadixSort::SortPairs(nullptr, tb, k0, k1, v0, v1, (int)np, 0, end_bit, s);
        if (e == cudaSuccess) e = cudaMallocAsync(&tmp, tb, s);
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(tmp, tb, k0, k1, v0, v1, (int)np, 0, end_bit, s);
    }
    if (e == cudaSuccess && n_rows) e = cudaMemsetAsync(row_version, 0, n_rows * 4, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_mixed, 0, 4, s);
    if (e == cudaSuccess) {
        tf_load_offsets_kernel<<<(uint32_t)((n_rows + 256) / 256), 256, 0, s>>>(k1, np, n_rows, st.d_row_off);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && np) {
        tf_load_rows_kernel<<<(uint32_t)((np + 255) / 256), 256, 0, s>>>(k1, v1, np, st.d_keys, st.d_vals, row_version, d_mixed);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    std::vector<uint64_t> row_off(n_rows + 1);
    std::vector<uint32_t> h_version(n_rows);
    uint32_t mixed = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(row_off.data(), st.d_row_off, (n_rows + 1) * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && n_rows) e = cudaMemcpyAsync(h_version.data(), row_version, n_rows * 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&mixed, d_mixed, 4, cudaMemcpyDeviceToHost, s);
    cdb_status rc = done(e);
    if (rc) return rc;
    CDB_REQUIRE(!mixed, "tf-idf load: a row's words carry two versions");
    // per-row state: a row with a live word counts, and so does a row the mask names; a 0 in the mask on such a row is refused
    std::vector<uint8_t> h_counted(n_rows);
    for (uint64_t r = 0; r < n_rows; ++r) {
        const bool words = row_off[r + 1] > row_off[r];
        CDB_REQUIRE(!counted || counted[r] || !words, "tf-idf load: counted is 0 for a row with live words");
        h_counted[r] = words || (counted && counted[r]) ? 1 : 0;
    }
    // the tiles; then the term table: the files' terms and df with carry_stats, else the hashes of the loaded pairs with df 0
    BuildBufs b;
    rc = b.alloc(std::max<uint64_t>(max_tile_pairs(row_off), carry ? 0 : np), TfCodec::END_BIT, s);
    if (!rc) rc = st.load_rows(std::move(row_off), b, s);
    if (rc) return rc;
    std::vector<uint32_t> terms, df;
    if (carry) {
        terms = f->hashes;
        df = f->df;
    } else {
        std::vector<uint32_t> cnt;
        if ((e = distinct_hashes(st.d_keys, np, b, s, terms, cnt)) != cudaSuccess) {
            set_error(std::string("tf-idf load: ") + cudaGetErrorString(e));
            return CDB_CUDA_ERROR;
        }
        df.assign(terms.size(), 0u);
    }
    const uint32_t docs = carry ? f->n_docs : 0u;
    if ((rc = upload_terms(ix, terms, df, docs, true, s))) return rc;
    ix->h_terms.swap(terms);
    ix->h_df.swap(df);
    ix->documents = docs;
    ix->version = f->max_version;
    ix->h_counted.swap(h_counted);
    ix->h_version.swap(h_version);
    return CDB_OK;
}

}  // namespace

namespace cdb {
int tfidf_index_device(const cdb_tfidf_index *ix) { return ix->desc.device; }

// ---------------------------------------------------------------- a shard group's TF-IDF search (shard_group.cu)
// Every function below runs on the caller's current device and stream; the ones taking an index expect its reader lock held.
std::shared_mutex &tfidf_index_mutex(cdb_tfidf_index *ix) { return ix->rw; }
uint32_t tfidf_index_id_base(const cdb_tfidf_index *ix) { return ix->desc.id_base; }
uint64_t tfidf_index_capacity(const cdb_tfidf_index *ix) { return ix->desc.capacity_rows; }
uint32_t tfidf_out_cols(uint32_t k) { return out_cols(k); }

// one shard's statistics for the group's idf, [N, df of d_qhash[0..n_qh)] as u32 at out (tf_query_stats_kernel)
cdb_status tfidf_shard_stats(const cdb_tfidf_index *ix, const uint32_t *d_qhash, uint64_t n_qh, uint32_t *out, cudaStream_t s) {
    tf_query_stats_kernel<<<(uint32_t)((n_qh + 256) / 256), 256, 0, s>>>(ix->d_terms, ix->d_df, (uint32_t)ix->h_terms.size(),
                                                                      ix->documents, d_qhash, n_qh, out);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// the group's idf of every query term into q_idf[0..n_qh) from the all-gathered statistics (rank r's at gathered + r * words)
cdb_status tfidf_group_idf(const uint64_t *gathered, size_t words, uint32_t world, uint64_t n_qh, float *q_idf, cudaStream_t s) {
    if (!n_qh) return CDB_OK;
    tf_group_idf_kernel<<<(uint32_t)((n_qh + 255) / 256), 256, 0, s>>>(gathered, words, world, n_qh, q_idf);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// one shard's half: every bucket winner of every query under the group's idf (d_qidf, one per query term) into out [nq][512].
// No term at or past n_qh is read.
cdb_status tfidf_shard_winners(cdb_tfidf_index *ix, const uint64_t *d_qoff, const uint32_t *d_qhash, uint64_t n_qh, const float *d_qidf,
                               uint32_t nq, uint2 *out, cudaStream_t s) {
    if (!nq) return CDB_OK;
    const uint32_t n_tiles = (uint32_t)ix->st.h_tiles.size();
    if (n_tiles == 0) {   // every bucket empty: id CDB_INVALID_ID
        CDB_CUDA_TRY(cudaMemsetAsync(out, 0xFF, (size_t)nq * TF_BUCKETS * sizeof(uint2), s));
        return CDB_OK;
    }
    size_t per_q = 0;
    const uint32_t chunk = score_chunk(nq, n_tiles, &per_q);
    uint2 *win = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&win, (size_t)chunk * per_q, s));
    cdb_status rc = CDB_OK;
    cudaError_t e = allow_max_dynamic_smem((const void *)tf_score_tile_kernel);
    if (e != cudaSuccess) { set_error(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    for (uint32_t q0 = 0; q0 < nq && !rc; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        tf_score_tile_kernel<<<dim3(n_tiles, c), TF_THREADS, TF_SCORE_SMEM, s>>>(score_args(ix, d_qoff, d_qhash, n_qh, d_qidf, q0, win));
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; break; }
        tf_winners_kernel<<<c, TF_THREADS, 0, s>>>(win, n_tiles, out + (size_t)q0 * TF_BUCKETS);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(win, s);
    return rc;
}

// the group's results from the all-gathered winners (rank r's [nq][512] at gathered + r * words)
cdb_status tfidf_group_finalize(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t k, uint32_t *ids, float *scores,
                                uint32_t *counts, cudaStream_t s) {
    if (!nq) return CDB_OK;
    tf_group_finalize_kernel<<<nq, TF_THREADS, 0, s>>>(reinterpret_cast<const uint2 *>(gathered), words, world, out_cols(k), ids, scores, counts);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}
}  // namespace cdb

extern "C" {

cdb_status cdb_tfidf_index_create(const cdb_tfidf_index_desc *desc, cdb_tfidf_index **out) {
    CDB_REQUIRE(desc && out, "null argument");
    *out = nullptr;
    std::unique_ptr<cdb_tfidf_index> ix(new cdb_tfidf_index());
    ix->desc = *desc;
    const cdb_status rc = ix->st.init(desc->device, desc->id_base, desc->capacity_rows, desc->capacity_pairs);
    if (rc) return rc;
    *out = ix.release();
    return CDB_OK;
}

cdb_status cdb_tfidf_index_destroy(cdb_tfidf_index *ix) {
    if (!ix) return CDB_OK;
    cudaSetDevice(ix->desc.device);
    cudaDeviceSynchronize();
    delete ix;
    return CDB_OK;
}

uint64_t cdb_tfidf_index_size(const cdb_tfidf_index *ix) { return ix ? ix->st.n_rows : 0; }

cdb_status cdb_tfidf_index_append(cdb_tfidf_index *ix, const uint64_t *row_offsets, const uint32_t *hashes, const float *tfs,
                                  const uint8_t *counted, uint64_t n, uint32_t version) {
    CDB_REQUIRE(ix, "null index");
    if (!n) return CDB_OK;
    cdb_status rc = check_csr(row_offsets, n, "row_offsets");
    if (rc) return rc;
    const uint64_t np = row_offsets[n];
    CDB_REQUIRE((hashes && tfs) || !np, "null pairs");
    CDB_REQUIRE(np < (1ull << 31), "a row tile or an append holds 2^31 pairs or more");   // the df count below takes an int
    uint32_t n_counted = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (!counted || counted[i]) ++n_counted;
        else CDB_REQUIRE(row_offsets[i + 1] == row_offsets[i], "an uncounted row must be empty");
    }
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(version >= ix->version, "version is older than the index's latest");
    // the scratch also holds the df count of the whole append; the drain covers searches reading the idf as well
    Append a;
    if ((rc = ix->st.prepare_append(row_offsets, hashes, tfs, n, np, "tf-idf append", a))) return rc;
    const cudaStream_t s = a.sg.s;
    BuildBufs &b = a.b;
    const uint32_t *d_hashes = ix->st.d_keys + a.p_old;
    // df increments: the distinct hashes of the appended pairs and how many rows hold each (rows never repeat a hash)
    std::vector<uint32_t> uniq, cnt;
    const cudaError_t e = distinct_hashes(d_hashes, np, b, s, uniq, cnt);
    if (e != cudaSuccess) { set_error(std::string("tf-idf append: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    // the merged term table
    std::vector<uint32_t> terms, df;
    terms.reserve(ix->h_terms.size() + uniq.size());
    df.reserve(ix->h_terms.size() + uniq.size());
    size_t i = 0, j = 0;
    while (i < ix->h_terms.size() || j < uniq.size()) {
        if (j == uniq.size() || (i < ix->h_terms.size() && ix->h_terms[i] < uniq[j])) { terms.push_back(ix->h_terms[i]); df.push_back(ix->h_df[i]); ++i; }
        else if (i == ix->h_terms.size() || uniq[j] < ix->h_terms[i]) { terms.push_back(uniq[j]); df.push_back(cnt[j]); ++j; }
        else { terms.push_back(ix->h_terms[i]); df.push_back(ix->h_df[i] + cnt[j]); ++i; ++j; }
    }
    const bool new_terms = terms.size() != ix->h_terms.size();
    // the tiles, then the idf of every term under the new N; if the upload fails the previous table goes back as well
    const uint32_t docs = ix->documents + n_counted;
    rc = ix->st.commit_append(a, [&]() -> cdb_status {
        const cdb_status r = upload_terms(ix, terms, df, docs, new_terms, s);
        if (r) {
            const std::string msg = cdb_last_error_string();
            upload_terms(ix, ix->h_terms, ix->h_df, ix->documents, true, s);
            set_error(msg);
        }
        return r;
    });
    if (rc) return rc;
    ix->h_terms.swap(terms);
    ix->h_df.swap(df);
    ix->documents = docs;
    ix->version = version;
    for (uint64_t r = 0; r < n; ++r) ix->h_counted.push_back(!counted || counted[r] ? 1 : 0);
    ix->h_version.resize(a.r_new, version);
    return CDB_OK;
}

cdb_status cdb_tfidf_index_load_files(cdb_tfidf_index *ix, const cdb_tfidf_files *files, uint64_t n_rows, const uint8_t *counted,
                                      int32_t carry_stats) {
    CDB_REQUIRE(ix && files, "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->st.n_rows == 0 && ix->h_terms.empty() && ix->documents == 0, "load_files needs an empty index");
    CDB_REQUIRE(n_rows <= ix->desc.capacity_rows, "n_rows exceeds capacity_rows");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    // searches already enqueued on other streams finish first
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    const cdb_status rc = load_locked(ix, files, n_rows, counted, carry_stats != 0, sg.s);
    if (rc && ix->st.n_rows) {
        const std::string msg = cdb_last_error_string();
        BuildBufs none;   // dropping every row builds no tile
        ix->st.restore_rows(0, none, sg.s);
        cudaStreamSynchronize(sg.s);
        set_error(msg);
    }
    return rc;
}

cdb_status cdb_tfidf_index_delete_rows(cdb_tfidf_index *ix, const uint32_t *rows, uint64_t n, uint32_t version) {
    CDB_REQUIRE(ix && (rows || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(version >= ix->version, "version is older than the index's latest");
    // fresh: the rows this call deletes (already deleted rows are left alone)
    return ix->st.mark_deleted(rows, n, [&](const std::vector<uint32_t> &fresh) -> cdb_status {
        // VersionedVec::delete of each of their terms: a delete in the insert's version removes the entry (df - 1), a later
        // one marks it and pushes a tombstone word (df + 1)
        std::vector<uint64_t> goff(fresh.size() + 1, 0);
        for (size_t i = 0; i < fresh.size(); ++i) goff[i + 1] = goff[i] + ix->st.h_row_off[fresh[i] + 1] - ix->st.h_row_off[fresh[i]];
        const uint64_t ng = goff.back();
        std::vector<uint32_t> gh(ng);
        StreamGuard sg;
        CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
        cudaStream_t s = sg.s;
        if (ng) {
            uint8_t *buf = nullptr;
            const size_t bytes = fresh.size() * 4 + goff.size() * 8 + ng * 4;
            CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
            uint64_t *d_off = reinterpret_cast<uint64_t *>(buf);
            uint32_t *d_rows = reinterpret_cast<uint32_t *>(d_off + goff.size());
            uint32_t *d_out = d_rows + fresh.size();
            cudaError_t e = cudaMemcpyAsync(d_off, goff.data(), goff.size() * 8, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_rows, fresh.data(), fresh.size() * 4, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) {
                tf_gather_rows_kernel<<<(uint32_t)((fresh.size() * 32 + 255) / 256), 256, 0, s>>>(ix->st.d_row_off, ix->st.d_keys, d_rows,
                                                                                              d_off, (uint32_t)fresh.size(), d_out);
                g_launch_count.fetch_add(1, std::memory_order_relaxed);
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = cudaMemcpyAsync(gh.data(), d_out, ng * 4, cudaMemcpyDeviceToHost, s);
            cudaFreeAsync(buf, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e != cudaSuccess) { set_error(std::string("tf-idf delete: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
        }
        std::vector<uint32_t> df = ix->h_df;
        uint32_t docs = ix->documents;
        for (size_t i = 0; i < fresh.size(); ++i) {
            const uint32_t r = fresh[i];
            if (!ix->h_counted[r]) continue;     // delete_embedding returns early for an embedding without text
            --docs;
            const uint32_t delta = ix->h_version[r] == version ? 0xFFFFFFFFu : 1u;
            for (uint64_t p = goff[i]; p < goff[i + 1]; ++p) {
                const size_t g = std::lower_bound(ix->h_terms.begin(), ix->h_terms.end(), gh[p]) - ix->h_terms.begin();
                df[g] += delta;
            }
        }
        // queued searches have drained (they read the idf)
        const cdb_status rc = upload_terms(ix, ix->h_terms, df, docs, false, s);
        if (rc) return rc;
        ix->h_df.swap(df);
        ix->documents = docs;
        ix->version = version;
        return CDB_OK;
    });
}

cdb_status cdb_tfidf_index_deleted_rows(const cdb_tfidf_index *ix, uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total) {
    CDB_REQUIRE(ix && (out || !n), "null argument");
    std::shared_lock<std::shared_mutex> lock(const_cast<cdb_tfidf_index *>(ix)->rw);
    return ix->st.deleted_rows(first, n, out, out_total);
}

cdb_status cdb_tfidf_index_term_stats(cdb_tfidf_index *ix, const uint32_t *hashes, uint64_t n, uint32_t *out_df, float *out_idf,
                                      uint32_t *out_documents_count) {
    CDB_REQUIRE(ix && (hashes || !n), "null argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    if (out_documents_count) *out_documents_count = ix->documents;
    if (!n) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    // the idf as the device holds it
    std::vector<float> idf(ix->h_terms.size());
    if (!idf.empty()) CDB_CUDA_TRY(cudaMemcpy(idf.data(), ix->d_idf, idf.size() * 4, cudaMemcpyDeviceToHost));
    for (uint64_t i = 0; i < n; ++i) {
        const size_t g = std::lower_bound(ix->h_terms.begin(), ix->h_terms.end(), hashes[i]) - ix->h_terms.begin();
        const bool found = g < ix->h_terms.size() && ix->h_terms[g] == hashes[i];
        if (out_df) out_df[i] = found ? ix->h_df[g] : 0u;
        if (out_idf) out_idf[i] = found ? idf[g] : std::nanf("");
    }
    return CDB_OK;
}

cdb_status cdb_tfidf_search_batch_device(cdb_tfidf_index *ix, const uint64_t *d_q_offsets, const uint32_t *d_q_hashes, uint32_t nq,
                                         uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts, void *stream) {
    CDB_REQUIRE(ix && (d_q_offsets || !nq) && (d_ids || !nq) && (d_scores || !nq) && (d_counts || !nq), "null argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    return search_locked(ix, d_q_offsets, d_q_hashes, nq, k, d_ids, d_scores, d_counts, (cudaStream_t)stream);
}

cdb_status cdb_tfidf_search_batch(cdb_tfidf_index *ix, const uint64_t *q_offsets, const uint32_t *q_hashes, uint32_t nq, uint32_t k,
                                  uint32_t *out_ids, float *out_scores, uint32_t *out_counts) {
    CDB_REQUIRE(ix && (out_ids || !nq) && (out_scores || !nq) && (out_counts || !nq), "null argument");
    if (!nq) return CDB_OK;
    cdb_status rc = check_csr(q_offsets, nq, "q_offsets");
    if (rc) return rc;
    const uint64_t nqh = q_offsets[nq];
    CDB_REQUIRE(q_hashes || !nqh, "null query hashes");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    const size_t kout = out_cols(k);
    const size_t bytes = (nq + 1) * 8 + (size_t)nq * kout * 8 + (size_t)nq * 4 + nqh * 4;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    uint64_t *d_off = reinterpret_cast<uint64_t *>(buf);
    uint32_t *d_ids = reinterpret_cast<uint32_t *>(d_off + nq + 1);
    float *d_scores = reinterpret_cast<float *>(d_ids + (size_t)nq * kout);
    uint32_t *d_counts = reinterpret_cast<uint32_t *>(d_scores + (size_t)nq * kout);
    uint32_t *d_qh = d_counts + nq;
    cudaError_t e = cudaMemcpyAsync(d_off, q_offsets, (nq + 1) * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nqh) e = cudaMemcpyAsync(d_qh, q_hashes, nqh * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) { set_error(std::string("cudaMemcpyAsync: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) rc = search_locked(ix, d_off, d_qh, nq, (uint32_t)k, d_ids, d_scores, d_counts, s);
    if (!rc) {
        e = cudaMemcpyAsync(out_ids, d_ids, (size_t)nq * kout * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_scores, d_scores, (size_t)nq * kout * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_counts, d_counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error(std::string("tf-idf search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(buf, s);
    return rc;
}

// the library's two copies of the idf arithmetic (bm25_idf.h): the device one as the idf kernels run it, and the same source
// compiled for the host, which no search runs
cdb_status cdb_debug_bm25(int32_t on_device, const float *x, uint64_t n, float *out_log1p, const uint32_t *n_docs, const uint32_t *df,
                          uint64_t n_pairs, float *out_idf, void *stream) {
    CDB_REQUIRE((x && out_log1p) || !n, "null argument");
    CDB_REQUIRE((n_docs && df && out_idf) || !n_pairs, "null argument");
    if (!on_device) {
        for (uint64_t i = 0; i < n; ++i) out_log1p[i] = bm25_log1pf(x[i]);
        for (uint64_t j = 0; j < n_pairs; ++j) out_idf[j] = bm25_idf(n_docs[j], df[j]);
        return CDB_OK;
    }
    if (!n && !n_pairs) return CDB_OK;
    const uint64_t blocks = std::min<uint64_t>((std::max(n, n_pairs) + 255) / 256, 4096);
    tf_debug_bm25_kernel<<<(uint32_t)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, out_log1p, n_docs, df, n_pairs, out_idf);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // extern "C"
