// sparse.cu -- the sparse inverted index (InvertedIndex, src/indexes/inverted/mod.rs) on the GPU: ingest, deletes, scoring
// of posting lists (SparseAnnQueryBasic::sequential_search, src/models/sparse_ann_query.rs:68-147), the raw-value re-rank
// (finalize_sparse_ann_results, inverted/mod.rs:331-381) and the values_upper_bound sampler (inverted/mod.rs:148-247).
//
// Layout (DESIGN.md section 8c).  The rows and posting tiles are a PostingTiles store (posting_tiles.cuh) keyed by dim, with
// packed u32 entries row_in_tile << 8 | key, sorted by key descending inside a segment.  A search scores one (query, tile)
// per CTA into shared-memory u32 accumulators plus a touched flag per row, selects the tile's top k*f touched rows exactly
// (radix select on (sim << 32) | ~id), merges the tile lists, then sorts (and re-ranks) the survivors.
#include <algorithm>
#include <cmath>
#include <memory>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <vector>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "kernels.h"
#include "posting_tiles.cuh"

namespace cdb {
namespace {

constexpr int SP_THREADS = 512;
constexpr uint32_t SP_QCHUNK = SP_THREADS;       // query pairs resolved per pass of the scoring kernel
constexpr uint32_t SP_MAX_K = 1024;
constexpr uint32_t SP_MAX_CAND = 5120;       // k * reranking_factor
constexpr uint32_t SP_MERGE_KEYS = 25600;    // keys a merge CTA holds in shared memory (200 KB)
constexpr uint32_t SP_MERGE_MAX_LISTS = 63;  // lists a merge CTA takes at once

// InvertedIndexNode::quantize (src/models/inverted_index.rs:168-172): an f32 divide then an f32 multiply (no FMA), clamp
// keeps NaN, the saturating `as u8` sends NaN to 0
__device__ inline uint32_t sparse_quantize(float v, float ub, uint32_t maxq) {
    float x = __fmul_rn(__fdiv_rn(v, ub), (float)maxq);
    const float m = (float)maxq;
    if (x < 0.0f) x = 0.0f;
    if (x > m) x = m;
    const uint32_t q = (x != x) ? 0u : (uint32_t)x;
    return q < maxq ? q : maxq;
}

// posting entries row_in_tile << 8 | key, sorted on dim << 8 | 255 - key: key-descending inside a dim's segment, so the
// keys >= etv of a low query value are a prefix of it.  A row may repeat a dim.
struct SparseCodec {
    using Entry = uint32_t;
    static constexpr int END_BIT = 40, SEG_SHIFT = 8;
    static constexpr const char *DUPLICATE_ERROR = nullptr;
    float ub;
    uint32_t maxq;
    __device__ SortPair encode(uint32_t dim, float v, uint32_t row) const {
        const uint32_t key = sparse_quantize(v, ub, maxq);
        return {((uint64_t)dim << 8) | (255u - key), (row << 8) | key};
    }
    __device__ Entry entry(uint64_t, uint32_t v) const { return v; }
};

// ---------------------------------------------------------------- search side
// Exact threshold of the top `need` keys among the non-zero keys key_at(0..n) (unique; more than `need` of them):
// keys >= the result are exactly the top `need`.  8-bit radix passes from the top, stopping once a bucket is taken whole.
template <class KeyAt>
__device__ uint64_t sp_select_threshold(uint32_t n, uint32_t need, KeyAt key_at, uint32_t *hist, uint32_t *state) {
    uint64_t prefix = 0;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (uint32_t i = tid; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const uint64_t hmask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        for (uint32_t i = tid; i < n; i += blockDim.x) {
            const uint64_t k = key_at(i);
            if (k && (k & hmask) == prefix) atomicAdd(&hist[(uint32_t)(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {
            uint32_t c[8], sum = 0;
#pragma unroll
            for (int s = 0; s < 8; ++s) { c[s] = hist[255 - 8 * lane - s]; sum += c[s]; }
            uint32_t incl = sum;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, off);
                if (lane >= (uint32_t)off) incl += t;
            }
            const uint32_t excl = incl - sum;
            if (excl < need && need <= incl) {
                uint32_t acc = excl;
                for (int s = 0; s < 8; ++s) {
                    if (acc + c[s] >= need) { state[0] = 255 - 8 * lane - s; state[1] = need - acc; state[2] = c[s]; break; }
                    acc += c[s];
                }
            }
        }
        __syncthreads();
        const uint32_t d = state[0], rem = state[1], bc = state[2];
        __syncthreads();
        prefix |= (uint64_t)d << shift;
        need = rem;
        if (rem == bc) break;
    }
    return prefix;
}

struct SpSearch {
    const uint32_t *entries, *tdims, *tseg, *deleted;
    const PostingTile *tiles;
    uint64_t n_rows;
    uint32_t id_base, maxq, etv, low;
    float ub;
    const uint64_t *q_off;
    const uint32_t *q_dims;
    const float *q_vals;
    uint32_t q0;            // first query of the chunk
    uint32_t m;             // candidates kept per query (k * factor)
    uint32_t n_tiles;
    uint64_t *out_keys;     // [chunk][n_tiles][m]
    uint32_t *out_cnt;      // [chunk][n_tiles]
};

constexpr size_t SP_SCORE_SMEM = (size_t)TILE_ROWS * 4 + TILE_ROWS + SP_QCHUNK * 8 + (SP_QCHUNK + 1) * 8 + SP_QCHUNK * 4 + 260 * 4;

__global__ void __launch_bounds__(SP_THREADS, 1) sp_score_tile_kernel(SpSearch a) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *acc = reinterpret_cast<uint32_t *>(smem);
    uint8_t *touched = smem + (size_t)TILE_ROWS * 4;
    uint64_t *c_beg = reinterpret_cast<uint64_t *>(touched + TILE_ROWS);
    uint64_t *c_pre = c_beg + SP_QCHUNK;
    uint32_t *c_qv = reinterpret_cast<uint32_t *>(c_pre + SP_QCHUNK + 1);
    uint32_t *hist = c_qv + SP_QCHUNK;   // 256 + state[4]
    using Scan = cub::BlockScan<unsigned long long, SP_THREADS>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ uint32_t s_cnt;

    const uint32_t t = blockIdx.x, qi = blockIdx.y, q = a.q0 + qi, tid = threadIdx.x;
    const PostingTile tile = a.tiles[t];
    const uint64_t row0 = (uint64_t)t << TILE_SHIFT;
    const uint32_t nr = (uint32_t)std::min<uint64_t>(TILE_ROWS, a.n_rows - row0);
    uint4 *a4 = reinterpret_cast<uint4 *>(acc);
    for (uint32_t i = tid; i < TILE_ROWS / 4; i += SP_THREADS) a4[i] = make_uint4(0, 0, 0, 0);
    uint4 *t4 = reinterpret_cast<uint4 *>(touched);
    for (uint32_t i = tid; i < TILE_ROWS / 16; i += SP_THREADS) t4[i] = make_uint4(0, 0, 0, 0);
    if (tid == 0) s_cnt = 0;
    __syncthreads();   // an empty query reaches the touched scan below without passing another barrier

    const uint32_t *tdims = a.tdims + tile.key_base;
    const uint32_t *tseg = a.tseg + tile.key_base + t;
    const uint32_t *ent = a.entries + tile.entry_base;
    const uint64_t qb = a.q_off[q], qe = a.q_off[q + 1];
    for (uint64_t j0 = qb; j0 < qe; j0 += SP_QCHUNK) {
        const uint32_t nj = (uint32_t)std::min<uint64_t>(SP_QCHUNK, qe - j0);
        unsigned long long len = 0;
        if (tid < nj) {
            const uint32_t d = a.q_dims[j0 + tid];
            const uint32_t qv = sparse_quantize(a.q_vals[j0 + tid], a.ub, a.maxq);
            const uint32_t lo = lower_bound_u32(tdims, tile.n_keys, d);
            uint32_t s = 0, e = 0;
            if (lo < tile.n_keys && tdims[lo] == d) {
                s = tseg[lo]; e = tseg[lo + 1];
                if (!(qv > a.low)) {                  // keys etv..=max only: a prefix of the key-descending segment
                    uint32_t l2 = s, h2 = e;
                    while (l2 < h2) { const uint32_t mid = (l2 + h2) >> 1; if ((ent[mid] & 255u) >= a.etv) l2 = mid + 1; else h2 = mid; }
                    e = l2;
                }
            }
            c_beg[tid] = s;
            c_qv[tid] = qv;
            len = e - s;
        }
        unsigned long long pre;
        Scan(scan_tmp).ExclusiveSum(len, pre);
        if (tid < nj) c_pre[tid] = pre;
        if (tid == nj - 1) c_pre[nj] = pre + len;
        __syncthreads();
        const unsigned long long total = c_pre[nj];
        uint32_t j = 0;
        for (unsigned long long i = tid; i < total; i += SP_THREADS) {
            while (c_pre[j + 1] <= i) ++j;
            const uint32_t e = __ldg(ent + c_beg[j] + (i - c_pre[j]));
            const uint32_t r = e >> 8;
            atomicAdd(&acc[r], c_qv[j] * (e & 255u));
            touched[r] = 1;
        }
        __syncthreads();
    }
    // deleted rows are never candidates; count the rest
    uint32_t mine = 0;
    for (uint32_t r = tid; r < nr; r += SP_THREADS) {
        if (!touched[r]) continue;
        const uint64_t g = row0 + r;
        if (a.deleted && (a.deleted[g >> 5] >> (g & 31)) & 1u) touched[r] = 0;
        else ++mine;
    }
    mine = __reduce_add_sync(0xFFFFFFFFu, mine);
    if ((tid & 31) == 0 && mine) atomicAdd(&s_cnt, mine);
    __syncthreads();
    const uint32_t nnz = s_cnt;
    const uint32_t id0 = a.id_base + (uint32_t)row0;
    auto key_at = [&](uint32_t r) -> uint64_t {
        return touched[r] ? (((uint64_t)acc[r] << 32) | (uint64_t)(~(id0 + r))) : 0ull;
    };
    const uint64_t thr = nnz > a.m ? sp_select_threshold(nr, a.m, key_at, hist, hist + 256) : 1ull;
    __syncthreads();
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    uint64_t *out = a.out_keys + ((size_t)qi * a.n_tiles + t) * a.m;
    for (uint32_t r = tid; r < nr; r += SP_THREADS) {
        const uint64_t k = key_at(r);
        if (k && k >= thr) out[atomicAdd(&s_cnt, 1u)] = k;
    }
    __syncthreads();
    if (tid == 0) a.out_cnt[(size_t)qi * a.n_tiles + t] = s_cnt;
}

// where the input lists of a merge live: list l of query qi is keys[qi * kq + l * kl ..] with cnt[qi * cq + l * cl] keys.
// The tree's own levels are [q][n_in][m] (kq = n_in * m, kl = m, cq = n_in, cl = 1); a shard group's gather buffer is
// rank-major, one list per rank (lists_rank_major).
struct SpLists {
    const uint64_t *keys;
    const uint32_t *cnt;
    size_t kq, kl, cq, cl;
};
inline SpLists lists_of_level(const uint64_t *keys, const uint32_t *cnt, uint32_t n_in, uint32_t m) {
    return {keys, cnt, (size_t)n_in * m, m, n_in, 1};
}

// lists -> [q][ceil(n_in / g)][m]: the top m of every group of g lists
__global__ void __launch_bounds__(SP_THREADS, 1) sp_merge_kernel(SpLists in, uint32_t n_in, uint32_t g, uint32_t m,
                                                                  uint64_t *__restrict__ out_keys, uint32_t *__restrict__ out_cnt) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    __shared__ uint32_t hist[260], s_off[SP_MERGE_MAX_LISTS + 1], s_cnt;
    const uint32_t grp = blockIdx.x, qi = blockIdx.y, tid = threadIdx.x, n_out = gridDim.x;
    const uint32_t l0 = grp * g, nl = min(g, n_in - l0);
    if (tid == 0) {
        uint32_t o = 0;
        for (uint32_t l = 0; l < nl; ++l) { s_off[l] = o; o += in.cnt[qi * in.cq + (l0 + l) * in.cl]; }
        s_off[nl] = o;
        s_cnt = 0;
    }
    __syncthreads();
    for (uint32_t l = 0; l < nl; ++l) {
        const uint64_t *src = in.keys + qi * in.kq + (l0 + l) * in.kl;
        for (uint32_t i = tid; i < s_off[l + 1] - s_off[l]; i += SP_THREADS) keys[s_off[l] + i] = src[i];
    }
    __syncthreads();
    const uint32_t n = s_off[nl];
    auto key_at = [&](uint32_t i) -> uint64_t { return keys[i]; };
    const uint64_t thr = n > m ? sp_select_threshold(n, m, key_at, hist, hist + 256) : 1ull;
    uint64_t *out = out_keys + ((size_t)qi * n_out + grp) * m;
    for (uint32_t i = tid; i < n; i += SP_THREADS) {
        const uint64_t k = keys[i];
        if (k >= thr) out[atomicAdd(&s_cnt, 1u)] = k;
    }
    __syncthreads();
    if (tid == 0) out_cnt[(size_t)qi * n_out + grp] = s_cnt;
}

// finalize_sparse_ann_results' dot product of one candidate row (pairs [rb, re)) with the query pairs [qb, qe), by one
// whole warp: the query pairs of a 32-wide chunk meet the row's pairs through shuffles (a row's later pair of a dim
// overwrites an earlier one, dims the row lacks are skipped), then dp = 0f32; dp += row_v * q_v sequentially in the
// caller's order.  Every lane returns dp.  Both re-ranks (sp_finalize_kernel, sp_rerank_all_kernel) call this.
__device__ __forceinline__ float sp_rerank_dot(uint64_t qb, uint64_t qe, const uint32_t *__restrict__ q_dims,
                                               const float *__restrict__ q_vals, uint64_t rb, uint64_t re,
                                               const uint32_t *__restrict__ dims, const float *__restrict__ vals) {
    const uint32_t lane = threadIdx.x & 31;
    float dp = 0.0f;
    for (uint64_t j0 = qb; j0 < qe; j0 += 32) {
        const uint32_t nj = (uint32_t)std::min<uint64_t>(32, qe - j0);
        uint32_t qd = 0xFFFFFFFFu;
        float qv = 0.0f, val = 0.0f;
        bool found = false;
        if (lane < nj) { qd = q_dims[j0 + lane]; qv = q_vals[j0 + lane]; }
        for (uint64_t p0 = rb; p0 < re; p0 += 32) {
            const uint32_t np = (uint32_t)std::min<uint64_t>(32, re - p0);
            uint32_t rd = 0;
            float rv = 0.0f;
            if (lane < np) { rd = dims[p0 + lane]; rv = vals[p0 + lane]; }
            for (uint32_t l = 0; l < np; ++l) {
                const uint32_t d = __shfl_sync(0xFFFFFFFFu, rd, l);
                const float v = __shfl_sync(0xFFFFFFFFu, rv, l);
                if (lane < nj && d == qd) { val = v; found = true; }
            }
        }
        for (uint32_t l = 0; l < nj; ++l) {
            const bool f = __shfl_sync(0xFFFFFFFFu, found, l);
            const float x = __shfl_sync(0xFFFFFFFFu, val, l), y = __shfl_sync(0xFFFFFFFFu, qv, l);
            if (f) dp = __fadd_rn(dp, __fmul_rn(x, y));
        }
    }
    return dp;
}

// the re-ranked selection key: total_cmp order of the canonicalised dp, then the smaller id
__device__ __forceinline__ uint64_t sp_rerank_key(float dp, uint32_t id) {
    return ((uint64_t)order_key(CDB_METRIC_DOT_PRODUCT, __float_as_uint(canon_nan(dp))) << 32) | (uint64_t)(~id);
}

// a selection key's score: the re-ranked f32, else the u32 similarity as f32
__device__ __forceinline__ float sp_key_score(uint64_t key, int rerank) {
    const uint32_t hi = (uint32_t)(key >> 32);
    return rerank ? __uint_as_float(key_to_bits(CDB_METRIC_DOT_PRODUCT, hi)) : __uint2float_rn(hi);
}

// one list of <= m candidates per query -> the best k, best first.  rerank: finalize_sparse_ann_results -- for every
// candidate dp = 0f32, dp += doc_val * q_val over the query pairs in the caller's order (a row's last pair of a dim wins),
// then total_cmp order (NaN canonicalised), ties to the smaller id.  Otherwise the score is the u32 similarity as f32.
// rerank = 2: the keys are already re-ranked (a shard group's combined list); sort and decode only.
__global__ void __launch_bounds__(SP_THREADS, 1) sp_finalize_kernel(const uint64_t *__restrict__ in_keys, const uint32_t *__restrict__ in_cnt,
                                                                     uint32_t m, uint32_t k, int rerank, uint32_t q0,
                                                                     const uint64_t *__restrict__ q_off, const uint32_t *__restrict__ q_dims,
                                                                     const float *__restrict__ q_vals, const uint64_t *__restrict__ row_off,
                                                                     const uint32_t *__restrict__ dims, const float *__restrict__ vals,
                                                                     uint32_t id_base, uint32_t *__restrict__ out_ids,
                                                                     float *__restrict__ out_scores, uint32_t *__restrict__ out_counts) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);   // pow2ceil(m) keys
    const uint32_t qi = blockIdx.x, q = q0 + qi, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n = in_cnt[qi];
    const uint64_t *src = in_keys + (size_t)qi * m;
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = tid; i < P; i += SP_THREADS) keys[i] = i < n ? src[i] : 0ull;
    __syncthreads();
    if (rerank == 1) {
        const uint64_t qb = q_off[q], qe = q_off[q + 1];
        for (uint32_t c = warp; c < n; c += SP_THREADS / 32) {
            const uint32_t id = ~(uint32_t)keys[c];
            const float dp = sp_rerank_dot(qb, qe, q_dims, q_vals, row_off[id - id_base], row_off[id - id_base + 1], dims, vals);
            if (lane == 0) keys[c] = sp_rerank_key(dp, id);
        }
        __syncthreads();
    }
    bitonic_sort<true>(keys, P);
    const uint32_t cnt = min(n, k);
    for (uint32_t i = tid; i < k; i += SP_THREADS) {
        uint32_t id = CDB_INVALID_ID;
        float s = 0.0f;
        if (i < cnt) {
            const uint64_t key = keys[i];
            id = ~(uint32_t)key;
            s = sp_key_score(key, rerank);
        }
        out_ids[(size_t)qi * k + i] = id;
        out_scores[(size_t)qi * k + i] = s;
    }
    if (tid == 0) out_counts[qi] = cnt;
}

// ---------------------------------------------------------------- top_k None: every candidate
// The scoring kernel runs with m = TILE_ROWS, so it never selects and writes every touched live row of (query qi, tile t)
// into slot [qi][t].  pos = exclusive scan of the [chunk][n_tiles] counts, so query qi's candidates become the contiguous
// segment [pos[qi * n_tiles], pos[(qi + 1) * n_tiles]).  One CTA per (tile, query) copies its slot there, tags each key with
// its query, and the (0, qi) CTA writes the segment offset seg[qi] (the last query's also seg[chunk]).
__global__ void __launch_bounds__(256) sp_all_gather_kernel(const uint64_t *__restrict__ slots, const uint32_t *__restrict__ cnt,
                                                            const uint32_t *__restrict__ pos, uint32_t n_tiles, uint64_t *__restrict__ keys,
                                                            uint32_t *__restrict__ qis, uint32_t *__restrict__ seg) {
    const uint32_t t = blockIdx.x, qi = blockIdx.y, slot = qi * n_tiles + t;
    const uint32_t n = cnt[slot], base = pos[slot];
    const uint64_t *src = slots + (size_t)slot * TILE_ROWS;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        keys[base + i] = src[i];
        qis[base + i] = qi;
    }
    if (t == 0 && threadIdx.x == 0) {
        seg[qi] = pos[slot];
        if (qi == gridDim.y - 1) seg[qi + 1] = pos[(qi + 1) * n_tiles];
    }
}

// rerank = 1 over the flat candidate array: one warp per candidate, the query from its tag, the same dot product as
// sp_finalize_kernel, rekeyed in place
__global__ void __launch_bounds__(256) sp_rerank_all_kernel(uint64_t *__restrict__ keys, const uint32_t *__restrict__ qis, uint32_t n,
                                                            uint32_t q0, const uint64_t *__restrict__ q_off, const uint32_t *__restrict__ q_dims,
                                                            const float *__restrict__ q_vals, const uint64_t *__restrict__ row_off,
                                                            const uint32_t *__restrict__ dims, const float *__restrict__ vals, uint32_t id_base) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t c = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n; c += warps) {
        const uint32_t id = ~(uint32_t)keys[c], q = q0 + qis[c];
        const float dp = sp_rerank_dot(q_off[q], q_off[q + 1], q_dims, q_vals, row_off[id - id_base], row_off[id - id_base + 1], dims, vals);
        if (lane == 0) keys[c] = sp_rerank_key(dp, id);
    }
}

// a shard group's phase 2: keys [nq][m] are the group's top m candidates per query (cnt[q] of them).  One warp per
// position: a candidate this shard owns (id_base <= id < id_base + n_rows) gets its re-ranked key from the same dot product
// as sp_finalize_kernel, every other position 0, so OR-ing the ranks' lists gives each candidate its key exactly once.
__global__ void __launch_bounds__(256) sp_rerank_owned_kernel(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ cnt, uint32_t nq,
                                                              uint32_t m, const uint64_t *__restrict__ q_off, const uint32_t *__restrict__ q_dims,
                                                              const float *__restrict__ q_vals, const uint64_t *__restrict__ row_off,
                                                              const uint32_t *__restrict__ dims, const float *__restrict__ vals, uint32_t id_base,
                                                              uint64_t n_rows, uint64_t *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5, n = (uint64_t)nq * m;
    for (uint64_t c = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n; c += warps) {
        const uint32_t q = (uint32_t)(c / m), j = (uint32_t)(c - (uint64_t)q * m);
        uint64_t key = 0;
        if (j < cnt[q]) {
            const uint32_t id = ~(uint32_t)keys[c], r = id - id_base;
            if (r < n_rows) key = sp_rerank_key(sp_rerank_dot(q_off[q], q_off[q + 1], q_dims, q_vals, row_off[r], row_off[r + 1], dims, vals), id);
        }
        if (lane == 0) out[c] = key;
    }
}

// out[i] = OR over the ranks of gathered[r * words + i]: the re-ranked lists of a shard group, one non-zero rank per position
__global__ void __launch_bounds__(256) sp_or_ranks_kernel(const uint64_t *__restrict__ gathered, size_t words, uint32_t world, uint64_t n,
                                                          uint64_t *__restrict__ out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t v = 0;
        for (uint32_t r = 0; r < world; ++r) v |= gathered[r * words + i];
        out[i] = v;
    }
}

// keys -> ids and scores, as sp_finalize_kernel writes them
__global__ void __launch_bounds__(256) sp_all_decode_kernel(const uint64_t *__restrict__ keys, uint32_t n, int rerank, uint32_t *__restrict__ ids,
                                                            float *__restrict__ scores) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t key = keys[i];
        ids[i] = ~(uint32_t)key;
        scores[i] = sp_key_score(key, rerank);
    }
}

// top_k None over a shard group: the ranks' sorted runs of one key sub-batch of nb queries -> the merged entries, decoded.
// gathered: rank r's keys at r * words, query j's run at pre[r * (nb + 1) + j] with pre[r * (nb + 1) + nb] - its start keys
// (an exclusive scan of the rank's counts).  The n entries are numbered rank after rank; each thread takes one, finds its
// rank and query, and writes it at its index in its run plus, for every rank, that rank's entries of the earlier queries
// and, for every other rank, the number of that rank's keys of the query greater than it (binary search; keys are unique
// across ranks).  One grid covers every entry of the sub-batch, however its queries' sizes are spread.
__global__ void __launch_bounds__(256) sp_merge_runs_all_kernel(const uint64_t *__restrict__ gathered, size_t words, uint32_t world,
                                                                const uint32_t *__restrict__ pre, uint32_t nb, uint32_t n, int rerank,
                                                                uint32_t *__restrict__ ids, float *__restrict__ scores) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint32_t r = 0, l = i;
        while (l >= pre[(size_t)r * (nb + 1) + nb]) { l -= pre[(size_t)r * (nb + 1) + nb]; ++r; }
        const uint32_t *P = pre + (size_t)r * (nb + 1);
        uint32_t lo = 0, hi = nb - 1;   // the query: the last j with P[j] <= l (P[nb] > l)
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (P[mid] <= l) lo = mid; else hi = mid - 1;
        }
        const uint32_t j = lo;
        const uint64_t key = gathered[(size_t)r * words + l];
        uint32_t pos = l;
        for (uint32_t o = 0; o < world; ++o) {
            if (o == r) continue;
            const uint32_t *O = pre + (size_t)o * (nb + 1);
            const uint64_t *R = gathered + (size_t)o * words;
            uint32_t b = O[j], e = O[j + 1];
            pos += b;
            while (b < e) {   // keys of rank o's run greater than `key`
                const uint32_t mid = (b + e) >> 1;
                if (R[mid] > key) b = mid + 1; else e = mid;
            }
            pos += b - O[j];
        }
        ids[pos] = ~(uint32_t)key;
        scores[pos] = sp_key_score(key, rerank);
    }
}

// sample_embedding: values > 1.0 ... > 9.0 (inverted/mod.rs:148-192)
__global__ void sp_sample_kernel(const float *__restrict__ v, uint64_t n, unsigned long long *__restrict__ counts) {
    uint32_t c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float x = __ldcs(v + i);
#pragma unroll
        for (int t = 0; t < 9; ++t) c[t] += x > (float)(t + 1);
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const uint32_t s = __reduce_add_sync(0xFFFFFFFFu, c[t]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(&counts[t], (unsigned long long)s);
    }
}

// Rust's `f32 as u32` / `as u8`: saturating, NaN -> 0
uint32_t sat_u32(float x, uint32_t hi) {
    if (!(x > 0.0f)) return 0;
    if (x >= (float)hi) return hi;
    return (uint32_t)x;
}

}  // namespace
}  // namespace cdb

using namespace cdb;

struct cdb_sparse_index {
    cdb_sparse_index_desc desc;
    std::shared_mutex rw;
    PostingTiles<SparseCodec> st;   // keys: dims
};

namespace {

cdb_status check_search_params(const cdb_sparse_search_params *p, uint32_t *m) {
    CDB_REQUIRE(p, "null params");
    CDB_REQUIRE(p->k >= 1 && p->k <= SP_MAX_K, "k must be in 1..1024");
    const uint64_t f = p->rerank ? p->reranking_factor : 1;
    CDB_REQUIRE(f >= 1 && (uint64_t)p->k * f <= SP_MAX_CAND, "k * reranking_factor must be in 1..5120");
    *m = (uint32_t)(p->k * f);
    return CDB_OK;
}

// sequential_search, sparse_ann_query.rs:80-83: etv = ((2^bits * thr).min(255.0)) as u8, low = (thr * 2^bits) as u32
void sp_thresholds(float thr, uint32_t bits, uint32_t *etv, uint32_t *low) {
    const float prod = (float)(1u << bits) * thr;
    const float etv_f = std::isnan(prod) ? 255.0f : std::min(prod, 255.0f);
    *etv = sat_u32(etv_f, 255);
    *low = sat_u32(thr * (float)(1u << bits), 0xFFFFFFFFu);
}

// the scoring kernel's arguments for queries [q0, q0 + chunk) keeping m candidates per (query, tile)
SpSearch score_args(const cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals,
                    const cdb_sparse_search_params *p, uint32_t q0, uint32_t m, uint64_t *out_keys, uint32_t *out_cnt) {
    const PostingTiles<SparseCodec> &st = ix->st;
    SpSearch a;
    a.entries = st.entries(); a.tdims = st.d_tkeys; a.tseg = st.d_tseg; a.deleted = st.deleted();
    a.tiles = st.d_tiles; a.n_rows = st.n_rows; a.id_base = ix->desc.id_base; a.maxq = st.codec.maxq;
    sp_thresholds(p->early_terminate_threshold, ix->desc.quantization_bits, &a.etv, &a.low);
    a.ub = st.codec.ub; a.q_off = d_qoff; a.q_dims = d_qdims; a.q_vals = d_qvals; a.q0 = q0; a.m = m;
    a.n_tiles = (uint32_t)st.h_tiles.size(); a.out_keys = out_keys; a.out_cnt = out_cnt;
    return a;
}

// the search on device buffers, under the reader lock
cdb_status search_locked(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                         const cdb_sparse_search_params *p, uint32_t m, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                         cudaStream_t s) {
    if (!nq) return CDB_OK;
    const uint32_t k = p->k;
    const uint32_t n_tiles = (uint32_t)ix->st.h_tiles.size();
    if (n_tiles == 0) return fill_empty_results(nq, k, d_ids, d_scores, d_counts, s);
    const uint32_t g = std::min<uint32_t>(SP_MERGE_MAX_LISTS, std::max<uint32_t>(2, SP_MERGE_KEYS / m));
    const uint32_t n_lvl1 = (n_tiles + g - 1) / g;
    uint32_t sort_cap = 1;
    while (sort_cap < m) sort_cap <<= 1;
    const size_t per_q = ((size_t)n_tiles + n_lvl1) * m * 8 + ((size_t)n_tiles + n_lvl1) * 4;
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)nq, 65535, (512ull << 20) / per_q}));
    uint64_t *ka = nullptr, *kb = nullptr;
    uint32_t *ca = nullptr, *cb = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&ka, (size_t)chunk * n_tiles * m * 8, s));
    cudaError_t e = cudaMallocAsync(&kb, (size_t)chunk * n_lvl1 * m * 8, s);
    if (e == cudaSuccess) e = cudaMallocAsync(&ca, (size_t)chunk * n_tiles * 4, s);
    if (e == cudaSuccess) e = cudaMallocAsync(&cb, (size_t)chunk * n_lvl1 * 4, s);
    cdb_status rc = CDB_OK;
    if (e != cudaSuccess) { set_error(std::string("cudaMallocAsync: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) {
        if ((e = allow_max_dynamic_smem((const void *)sp_score_tile_kernel)) != cudaSuccess ||
            (e = allow_max_dynamic_smem((const void *)sp_merge_kernel)) != cudaSuccess ||
            (e = allow_max_dynamic_smem((const void *)sp_finalize_kernel)) != cudaSuccess) {
            set_error(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e));
            rc = CDB_CUDA_ERROR;
        }
    }
    for (uint32_t q0 = 0; q0 < nq && !rc; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        const SpSearch a = score_args(ix, d_qoff, d_qdims, d_qvals, p, q0, m, ka, ca);
        sp_score_tile_kernel<<<dim3(n_tiles, c), SP_THREADS, SP_SCORE_SMEM, s>>>(a);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; break; }
        uint64_t *cur = ka, *nxt = kb;
        uint32_t *ccur = ca, *cnxt = cb, n_lists = n_tiles;
        while (n_lists > 1) {
            const uint32_t n_out = (n_lists + g - 1) / g;
            const uint32_t held = std::min<uint32_t>(g, n_lists) * m;
            sp_merge_kernel<<<dim3(n_out, c), SP_THREADS, (size_t)held * 8, s>>>(lists_of_level(cur, ccur, n_lists, m), n_lists, g, m,
                                                                                  nxt, cnxt);
            g_launch_count.fetch_add(1, std::memory_order_relaxed);
            if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; break; }
            std::swap(cur, nxt);
            std::swap(ccur, cnxt);
            n_lists = n_out;
        }
        if (rc) break;
        sp_finalize_kernel<<<c, SP_THREADS, (size_t)sort_cap * 8, s>>>(cur, ccur, m, k, p->rerank ? 1 : 0, q0, d_qoff, d_qdims, d_qvals, ix->st.d_row_off,
                                                    ix->st.d_keys, ix->st.d_vals, ix->desc.id_base, d_ids + (size_t)q0 * k,
                                                    d_scores + (size_t)q0 * k, d_counts + q0);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    for (void *ptr : {(void *)ka, (void *)kb, (void *)ca, (void *)cb})
        if (ptr) cudaFreeAsync(ptr, s);
    return rc;
}

// The top m keys of n_lists lists per query, for c queries, into dest_keys [c][m] / dest_cnt [c], unsorted: the merge tree
// of search_locked, whose last level writes the destination.  At least one level runs, so a single list is copied.
cdb_status merge_lists(SpLists in, uint32_t n_lists, uint32_t c, uint32_t m, uint64_t *dest_keys, uint32_t *dest_cnt, cudaStream_t s) {
    const uint32_t g = std::min<uint32_t>(SP_MERGE_MAX_LISTS, std::max<uint32_t>(2, SP_MERGE_KEYS / m));
    const uint32_t n1 = (n_lists + g - 1) / g;
    uint64_t *bk[2] = {nullptr, nullptr};
    uint32_t *bc[2] = {nullptr, nullptr};
    cdb_status rc = CDB_OK;
    cudaError_t e = allow_max_dynamic_smem((const void *)sp_merge_kernel);
    for (int i = 0; i < 2 && n1 > 1 && e == cudaSuccess; ++i) {
        e = cudaMallocAsync(&bk[i], (size_t)c * n1 * m * 8, s);
        if (e == cudaSuccess) e = cudaMallocAsync(&bc[i], (size_t)c * n1 * 4, s);
    }
    if (e != cudaSuccess) { set_error(std::string("sparse merge: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    for (uint32_t n = n_lists, w = 0; !rc; w ^= 1) {
        const uint32_t n_out = (n + g - 1) / g;
        uint64_t *ok = n_out == 1 ? dest_keys : bk[w];
        uint32_t *oc = n_out == 1 ? dest_cnt : bc[w];
        sp_merge_kernel<<<dim3(n_out, c), SP_THREADS, (size_t)std::min(g, n) * m * 8, s>>>(in, n, g, m, ok, oc);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
        in = lists_of_level(ok, oc, n_out, m);
        n = n_out;
        if (n == 1) break;
    }
    for (int i = 0; i < 2; ++i) {
        if (bk[i]) cudaFreeAsync(bk[i], s);
        if (bc[i]) cudaFreeAsync(bc[i], s);
    }
    return rc;
}

constexpr size_t SP_ALL_BUDGET = 512ull << 20;   // device scratch of one chunk of a top_k None search

// Sorts each query's segment of keys descending: a stable radix sort of all keys descending carrying their query tags,
// then a stable sort on the tags (qbits wide; none for a single query) carrying the keys.  Keys are unique per query.
cudaError_t sp_sort_segments(void *tmp, size_t tmp_bytes, cub::DoubleBuffer<uint64_t> &keys, cub::DoubleBuffer<uint32_t> &qis, uint32_t n,
                             int qbits, cudaStream_t s) {
    size_t tb = tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairsDescending(tmp, tb, keys, qis, (int)n, 0, 64, s);
    if (e == cudaSuccess && qbits) {
        tb = tmp_bytes;
        e = cub::DeviceRadixSort::SortPairs(tmp, tb, qis, keys, (int)n, 0, qbits, s);
    }
    return e;
}

int qbits_of(uint32_t c) { return c > 1 ? 32 - __builtin_clz(c - 1) : 0; }

// The top_k None search on device queries, under the reader lock: every candidate of every query, sorted (and re-ranked),
// appended to r in host memory.  Per chunk: the device half (sparse_all_keys), decode, copy out.
cdb_status search_all_locked(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                             const cdb_sparse_search_params *p, cdb_sparse_results *r, cudaStream_t s) {
    const PostingTiles<SparseCodec> &st = ix->st;
    const uint64_t n_live = st.n_rows - st.n_deleted;   // a query's candidates, at most
    r->off.assign((size_t)nq + 1, 0);
    if (!nq || st.h_tiles.empty() || !n_live) return CDB_OK;
    CDB_REQUIRE(n_live < (1ull << 31), "top_k None: an index with 2^31 live rows or more");
    SparseAllScratch sc;
    cdb_status rc = sparse_all_alloc(ix, sparse_all_chunk(nq, st.h_tiles.size(), n_live), &sc, s);
    auto run_chunk = [&](uint32_t q0, uint32_t c) -> cdb_status {
        cdb_status rc = sparse_all_keys(ix, d_qoff, d_qdims, d_qvals, p, q0, c, &sc, s);
        if (rc) return rc;
        const uint32_t total = sc.seg_h[c];
        const uint64_t base = r->ids.size();
        for (uint32_t i = 0; i < c; ++i) r->off[(size_t)q0 + i + 1] = base + sc.seg_h[i + 1];
        if (!total) return CDB_OK;
        uint32_t *ids = reinterpret_cast<uint32_t *>(sc.spare);   // the free half of the key buffers holds ids, then scores
        float *scores = reinterpret_cast<float *>(ids + total);
        sp_all_decode_kernel<<<std::min<uint32_t>((total + 255) / 256, 1u << 16), 256, 0, s>>>(sc.keys, total, p->rerank ? 1 : 0, ids, scores);
        CDB_LAUNCH_CHECK();
        r->ids.resize(base + total);
        r->scores.resize(base + total);
        CDB_CUDA_TRY(cudaMemcpyAsync(r->ids.data() + base, ids, (size_t)total * 4, cudaMemcpyDeviceToHost, s));
        CDB_CUDA_TRY(cudaMemcpyAsync(r->scores.data() + base, scores, (size_t)total * 4, cudaMemcpyDeviceToHost, s));
        CDB_CUDA_TRY(cudaStreamSynchronize(s));
        return CDB_OK;
    };
    try {
        for (uint32_t q0 = 0; q0 < nq && !rc; q0 += sc.chunk) rc = run_chunk(q0, std::min(sc.chunk, nq - q0));
    } catch (const std::bad_alloc &) {
        set_error("top_k None: host allocation of the results failed");
        rc = CDB_CUDA_ERROR;
    }
    sparse_all_free(&sc, s);
    return rc;
}

}  // namespace

namespace cdb {
cdb_status sparse_index_room(cdb_sparse_index *ix, uint64_t *rows, uint64_t *rows_left, uint64_t *pairs_left) {
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    *rows = ix->st.n_rows;
    *rows_left = ix->desc.capacity_rows - ix->st.n_rows;
    *pairs_left = ix->desc.capacity_pairs - ix->st.n_pairs;
    return CDB_OK;
}

cdb_status sparse_index_truncate(cdb_sparse_index *ix, uint64_t rows) {
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    PostingTiles<SparseCodec> &st = ix->st;
    CDB_REQUIRE(rows <= st.n_rows, "truncate beyond the index");
    if (rows == st.n_rows) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint64_t r0 = rows & ~(uint64_t)(TILE_ROWS - 1);
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    BuildBufs b;
    cdb_status rc = b.alloc(st.h_row_off[rows] - st.h_row_off[r0], SparseCodec::END_BIT, sg.s);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    return st.restore_rows(rows, b, sg.s);
}

int sparse_index_device(const cdb_sparse_index *ix) { return ix->desc.device; }

// ---------------------------------------------------------------- a shard group's sparse search (shard_group.cu)
// Every function below runs on the caller's current device and stream; the ones taking an index expect its reader lock held.
std::shared_mutex &sparse_index_mutex(cdb_sparse_index *ix) { return ix->rw; }
uint32_t sparse_index_bits(const cdb_sparse_index *ix) { return ix->desc.quantization_bits; }
float sparse_index_upper_bound(const cdb_sparse_index *ix) { return ix->desc.values_upper_bound; }
uint32_t sparse_index_id_base(const cdb_sparse_index *ix) { return ix->desc.id_base; }
uint64_t sparse_index_capacity(const cdb_sparse_index *ix) { return ix->desc.capacity_rows; }
cdb_status sparse_check_params(const cdb_sparse_search_params *p, uint32_t *m) { return check_search_params(p, m); }

// phase 1 on one shard: its top m candidates per query (the list sp_finalize_kernel would take), unsorted, into
// keys [nq][m] / cnt [nq]
cdb_status sparse_shard_select(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                               const cdb_sparse_search_params *p, uint32_t m, uint64_t *keys, uint32_t *cnt, cudaStream_t s) {
    const uint32_t n_tiles = (uint32_t)ix->st.h_tiles.size();
    if (!nq) return CDB_OK;
    if (!n_tiles) { CDB_CUDA_TRY(cudaMemsetAsync(cnt, 0, (size_t)nq * 4, s)); return CDB_OK; }
    const size_t per_q = (size_t)n_tiles * m * 12;
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)nq, 65535, (512ull << 20) / per_q}));
    uint64_t *ka = nullptr;
    uint32_t *ca = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&ka, (size_t)chunk * n_tiles * m * 8, s));
    cudaError_t e = cudaMallocAsync(&ca, (size_t)chunk * n_tiles * 4, s);
    if (e == cudaSuccess) e = allow_max_dynamic_smem((const void *)sp_score_tile_kernel);
    cdb_status rc = CDB_OK;
    if (e != cudaSuccess) { set_error(std::string("sparse shard search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    for (uint32_t q0 = 0; q0 < nq && !rc; q0 += chunk) {
        const uint32_t c = std::min(chunk, nq - q0);
        sp_score_tile_kernel<<<dim3(n_tiles, c), SP_THREADS, SP_SCORE_SMEM, s>>>(score_args(ix, d_qoff, d_qdims, d_qvals, p, q0, m, ka, ca));
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; break; }
        rc = merge_lists(lists_of_level(ka, ca, n_tiles, m), n_tiles, c, m, keys + (size_t)q0 * m, cnt + q0, s);
    }
    if (ka) cudaFreeAsync(ka, s);
    if (ca) cudaFreeAsync(ca, s);
    return rc;
}

// the group's top m per query from the all-gathered phase-1 lists: rank r's slot is gathered[r * words ..], keys [nq][m]
// then the u32 counts [nq]
cdb_status sparse_group_select(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t m, uint64_t *keys,
                               uint32_t *cnt, cudaStream_t s) {
    const SpLists in{gathered, reinterpret_cast<const uint32_t *>(gathered + (size_t)nq * m), m, words, 1, 2 * words};
    return merge_lists(in, world, nq, m, keys, cnt, s);
}

// phase 2 on one shard: out [nq][m] = the re-ranked key of every candidate of keys / cnt this shard owns, 0 elsewhere
cdb_status sparse_shard_rerank(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals, uint32_t nq,
                               uint32_t m, const uint64_t *keys, const uint32_t *cnt, uint64_t *out, cudaStream_t s) {
    const uint64_t n = (uint64_t)nq * m;
    if (!n) return CDB_OK;
    const uint32_t blocks = (uint32_t)std::min<uint64_t>((n + 7) / 8, 1u << 20);
    sp_rerank_owned_kernel<<<blocks, 256, 0, s>>>(keys, cnt, nq, m, d_qoff, d_qdims, d_qvals, ix->st.d_row_off, ix->st.d_keys, ix->st.d_vals,
                                                  ix->desc.id_base, ix->st.n_rows, out);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// the group's results: rerank = 0 sorts the top-k keys / cnt and scores them by similarity; rerank = 1 first ORs the
// ranks' phase-2 lists (gathered, rank r at r * words) into keys, then sorts the re-ranked keys.  Best k per query.
cdb_status sparse_group_finalize(const uint64_t *gathered, size_t words, uint32_t world, uint32_t nq, uint32_t m, uint32_t k, int rerank,
                                 uint64_t *keys, const uint32_t *cnt, uint32_t *ids, float *scores, uint32_t *counts, cudaStream_t s) {
    if (!nq) return CDB_OK;
    if (rerank) {
        const uint64_t n = (uint64_t)nq * m;
        sp_or_ranks_kernel<<<(uint32_t)std::min<uint64_t>((n + 255) / 256, 1u << 16), 256, 0, s>>>(gathered, words, world, n, keys);
        CDB_LAUNCH_CHECK();
    }
    uint32_t sort_cap = 1;
    while (sort_cap < m) sort_cap <<= 1;
    CDB_CUDA_TRY(allow_max_dynamic_smem((const void *)sp_finalize_kernel));
    sp_finalize_kernel<<<nq, SP_THREADS, (size_t)sort_cap * 8, s>>>(keys, cnt, m, k, rerank ? 2 : 0, 0, nullptr, nullptr, nullptr, nullptr,
                                                                     nullptr, nullptr, 0, ids, scores, counts);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// ---------------------------------------------------------------- the device half of a top_k None search
void sparse_index_all_bounds(const cdb_sparse_index *ix, uint64_t *n_tiles, uint64_t *n_live) {
    *n_tiles = ix->st.h_tiles.size();
    *n_live = ix->st.n_rows - ix->st.n_deleted;
}

uint32_t sparse_all_chunk(uint32_t nq, uint64_t n_tiles, uint64_t n_live) {
    const size_t per_q = (size_t)n_tiles * TILE_ROWS * 8 + (size_t)n_tiles * 8 + n_live * 24;
    return (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)nq, 65535, SP_ALL_BUDGET / std::max<size_t>(per_q, 1)}));
}

// nothing is allocated for an index without tiles or live rows: sparse_all_keys gives it no candidates
cdb_status sparse_all_alloc(cdb_sparse_index *ix, uint32_t chunk, SparseAllScratch *sc, cudaStream_t s) {
    const PostingTiles<SparseCodec> &st = ix->st;
    const uint32_t n_tiles = (uint32_t)st.h_tiles.size();
    const uint64_t n_live = st.n_rows - st.n_deleted;
    sc->chunk = chunk;
    sc->seg_h.assign((size_t)chunk + 1, 0);
    if (!n_tiles || !n_live) return CDB_OK;
    const uint64_t cap = (uint64_t)chunk * n_live;      // candidates of a chunk, at most (< 2^31: budget or one query)
    const uint32_t n_slots = chunk * n_tiles;
    size_t t_scan = 0, t_sort1 = 0, t_sort2 = 0;
    cub::DoubleBuffer<uint64_t> kd(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> qd(nullptr, nullptr);
    CDB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, sc->cnt, sc->pos, (int)n_slots + 1, s));
    CDB_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(nullptr, t_sort1, kd, qd, (int)cap, 0, 64, s));
    if (chunk > 1) CDB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t_sort2, qd, kd, (int)cap, 0, qbits_of(chunk), s));
    sc->tmp_bytes = std::max({t_scan, t_sort1, t_sort2});
    CDB_CUDA_TRY(cudaMallocAsync(&sc->slots, (size_t)n_slots * TILE_ROWS * 8, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->cnt, ((size_t)n_slots + 1) * 4, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->pos, ((size_t)n_slots + 1) * 4, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->seg, ((size_t)chunk + 1) * 4, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->ka, cap * 8, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->kb, cap * 8, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->qa, cap * 4, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->qb, cap * 4, s));
    CDB_CUDA_TRY(cudaMallocAsync(&sc->tmp, std::max<size_t>(sc->tmp_bytes, 1), s));
    CDB_CUDA_TRY(allow_max_dynamic_smem((const void *)sp_score_tile_kernel));
    return CDB_OK;
}

void sparse_all_free(SparseAllScratch *sc, cudaStream_t s) {
    for (void *ptr : {(void *)sc->slots, (void *)sc->cnt, (void *)sc->pos, (void *)sc->seg, (void *)sc->ka, (void *)sc->kb, (void *)sc->qa,
                      (void *)sc->qb, sc->tmp})
        if (ptr) cudaFreeAsync(ptr, s);
    *sc = SparseAllScratch();
}

// Queries [q0, q0 + c), c <= sc->chunk: score into per-(query, tile) slots, scan the slot counts, gather each query's keys into
// one segment, sort the segments, re-rank and sort again.  Waits for the stream once, to size the sort.
cdb_status sparse_all_keys(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals,
                           const cdb_sparse_search_params *p, uint32_t q0, uint32_t c, SparseAllScratch *sc, cudaStream_t s) {
    const PostingTiles<SparseCodec> &st = ix->st;
    const uint32_t n_tiles = (uint32_t)st.h_tiles.size();
    sc->keys = sc->spare = nullptr;
    if (!sc->slots) {   // no tiles or no live rows
        std::fill(sc->seg_h.begin(), sc->seg_h.begin() + c + 1, 0u);
        return CDB_OK;
    }
    const SpSearch a = score_args(ix, d_qoff, d_qdims, d_qvals, p, q0, TILE_ROWS, sc->slots, sc->cnt);
    sp_score_tile_kernel<<<dim3(n_tiles, c), SP_THREADS, SP_SCORE_SMEM, s>>>(a);
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaMemsetAsync(sc->cnt + (size_t)c * n_tiles, 0, 4, s));
    size_t tb = sc->tmp_bytes;
    CDB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(sc->tmp, tb, sc->cnt, sc->pos, (int)(c * n_tiles) + 1, s));
    sp_all_gather_kernel<<<dim3(n_tiles, c), 256, 0, s>>>(sc->slots, sc->cnt, sc->pos, n_tiles, sc->ka, sc->qa, sc->seg);
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->seg_h.data(), sc->seg, ((size_t)c + 1) * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    const uint32_t total = sc->seg_h[c];
    if (!total) return CDB_OK;
    cub::DoubleBuffer<uint64_t> kd(sc->ka, sc->kb);
    cub::DoubleBuffer<uint32_t> qd(sc->qa, sc->qb);
    CDB_CUDA_TRY(sp_sort_segments(sc->tmp, sc->tmp_bytes, kd, qd, total, qbits_of(c), s));
    if (p->rerank) {
        const uint32_t blocks = (uint32_t)std::min<uint64_t>(((uint64_t)total + 7) / 8, 1u << 20);
        sp_rerank_all_kernel<<<blocks, 256, 0, s>>>(kd.Current(), qd.Current(), total, q0, d_qoff, d_qdims, d_qvals, st.d_row_off,
                                                    st.d_keys, st.d_vals, ix->desc.id_base);
        CDB_LAUNCH_CHECK();
        CDB_CUDA_TRY(sp_sort_segments(sc->tmp, sc->tmp_bytes, kd, qd, total, qbits_of(c), s));
    }
    sc->keys = kd.Current();
    sc->spare = kd.Alternate();
    return CDB_OK;
}

// a shard group's top_k None merge of one key sub-batch (sp_merge_runs_all_kernel); d_pre as the kernel takes it
cdb_status sparse_group_merge_all(const uint64_t *gathered, size_t words, uint32_t world, const uint32_t *d_pre, uint32_t nb, uint32_t n,
                                  int rerank, uint32_t *ids, float *scores, cudaStream_t s) {
    if (!n) return CDB_OK;
    sp_merge_runs_all_kernel<<<std::min<uint32_t>((n + 255) / 256, 1u << 16), 256, 0, s>>>(gathered, words, world, d_pre, nb, n, rerank,
                                                                                             ids, scores);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}
}  // namespace cdb

extern "C" {

cdb_status cdb_sparse_index_create(const cdb_sparse_index_desc *desc, cdb_sparse_index **out) {
    CDB_REQUIRE(desc && out, "null argument");
    CDB_REQUIRE(desc->quantization_bits >= 4 && desc->quantization_bits <= 8, "quantization_bits must be in 4..8");
    *out = nullptr;
    std::unique_ptr<cdb_sparse_index> ix(new cdb_sparse_index());
    ix->desc = *desc;
    ix->st.codec = SparseCodec{desc->values_upper_bound, (1u << desc->quantization_bits) - 1};
    const cdb_status rc = ix->st.init(desc->device, desc->id_base, desc->capacity_rows, desc->capacity_pairs);
    if (rc) return rc;
    *out = ix.release();
    return CDB_OK;
}

cdb_status cdb_sparse_index_destroy(cdb_sparse_index *ix) {
    if (!ix) return CDB_OK;
    cudaSetDevice(ix->desc.device);
    cudaDeviceSynchronize();
    delete ix;
    return CDB_OK;
}

uint64_t cdb_sparse_index_size(const cdb_sparse_index *ix) { return ix ? ix->st.n_rows : 0; }

cdb_status cdb_sparse_index_append(cdb_sparse_index *ix, const uint64_t *row_offsets, const uint32_t *dims, const float *values,
                                   uint64_t n) {
    CDB_REQUIRE(ix, "null index");
    if (!n) return CDB_OK;
    cdb_status rc = check_csr(row_offsets, n, "row_offsets");
    if (rc) return rc;
    const uint64_t np = row_offsets[n];
    CDB_REQUIRE((dims && values) || !np, "null pairs");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    Append a;
    if ((rc = ix->st.prepare_append(row_offsets, dims, values, n, 0, "sparse append", a))) return rc;
    return ix->st.commit_append(a, [] { return CDB_OK; });
}

cdb_status cdb_sparse_index_delete_rows(cdb_sparse_index *ix, const uint32_t *rows, uint64_t n) {
    CDB_REQUIRE(ix && (rows || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    return ix->st.mark_deleted(rows, n, [](const std::vector<uint32_t> &) { return CDB_OK; });
}

cdb_status cdb_sparse_index_deleted_rows(const cdb_sparse_index *ix, uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total) {
    CDB_REQUIRE(ix && (out || !n), "null argument");
    std::shared_lock<std::shared_mutex> lock(const_cast<cdb_sparse_index *>(ix)->rw);
    return ix->st.deleted_rows(first, n, out, out_total);
}

cdb_status cdb_sparse_search_batch_device(cdb_sparse_index *ix, const uint64_t *d_q_offsets, const uint32_t *d_q_dims,
                                          const float *d_q_values, uint32_t nq, const cdb_sparse_search_params *p,
                                          uint32_t *d_ids, float *d_scores, uint32_t *d_counts, void *stream) {
    CDB_REQUIRE(ix && (d_q_offsets || !nq) && (d_ids || !nq) && (d_scores || !nq) && (d_counts || !nq), "null argument");
    uint32_t m = 0;
    cdb_status rc = check_search_params(p, &m);
    if (rc) return rc;
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    return search_locked(ix, d_q_offsets, d_q_dims, d_q_values, nq, p, m, d_ids, d_scores, d_counts, (cudaStream_t)stream);
}

cdb_status cdb_sparse_search_batch(cdb_sparse_index *ix, const uint64_t *q_offsets, const uint32_t *q_dims, const float *q_values,
                                   uint32_t nq, const cdb_sparse_search_params *p, uint32_t *out_ids, float *out_scores,
                                   uint32_t *out_counts) {
    CDB_REQUIRE(ix && (out_ids || !nq) && (out_scores || !nq) && (out_counts || !nq), "null argument");
    uint32_t m = 0;
    cdb_status rc = check_search_params(p, &m);
    if (rc) return rc;
    if (!nq) return CDB_OK;
    if ((rc = check_csr(q_offsets, nq, "q_offsets"))) return rc;
    const uint64_t nqp = q_offsets[nq];
    CDB_REQUIRE((q_dims && q_values) || !nqp, "null query pairs");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    const size_t k = p->k;
    const size_t bytes = (nq + 1) * 8 + nqp * 8 + (size_t)nq * k * 8 + (size_t)nq * 4;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    uint64_t *d_off = reinterpret_cast<uint64_t *>(buf);
    uint32_t *d_ids = reinterpret_cast<uint32_t *>(d_off + nq + 1);
    float *d_scores = reinterpret_cast<float *>(d_ids + (size_t)nq * k);
    uint32_t *d_counts = reinterpret_cast<uint32_t *>(d_scores + (size_t)nq * k);
    uint32_t *d_qd = d_counts + nq;
    float *d_qv = reinterpret_cast<float *>(d_qd + nqp);
    cudaError_t e = cudaMemcpyAsync(d_off, q_offsets, (nq + 1) * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nqp) e = cudaMemcpyAsync(d_qd, q_dims, nqp * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nqp) e = cudaMemcpyAsync(d_qv, q_values, nqp * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) { set_error(std::string("cudaMemcpyAsync: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) rc = search_locked(ix, d_off, d_qd, d_qv, nq, p, m, d_ids, d_scores, d_counts, s);
    if (!rc) {
        e = cudaMemcpyAsync(out_ids, d_ids, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_scores, d_scores, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_counts, d_counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error(std::string("sparse search: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    cudaFreeAsync(buf, s);
    return rc;
}

cdb_status cdb_sparse_search_batch_all(cdb_sparse_index *ix, const uint64_t *q_offsets, const uint32_t *q_dims, const float *q_values,
                                       uint32_t nq, const cdb_sparse_search_params *p, cdb_sparse_results **out) {
    CDB_REQUIRE(ix && p && out, "null argument");
    *out = nullptr;
    CDB_REQUIRE(p->k == 0, "cdb_sparse_search_batch_all takes k = 0 (top_k None)");
    uint64_t nqp = 0;
    if (nq) {
        const cdb_status rc = check_csr(q_offsets, nq, "q_offsets");
        if (rc) return rc;
        nqp = q_offsets[nq];
        CDB_REQUIRE((q_dims && q_values) || !nqp, "null query pairs");
    }
    std::unique_ptr<cdb_sparse_results> r(new (std::nothrow) cdb_sparse_results());
    CDB_REQUIRE(r, "out of host memory");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    if (!nq || ix->st.h_tiles.empty()) {   // no query or no row: every query has no candidate, nothing runs on the device
        r->off.assign((size_t)nq + 1, 0);
        *out = r.release();
        return CDB_OK;
    }
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    const size_t bytes = ((size_t)nq + 1) * 8 + nqp * 8;
    uint8_t *buf = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&buf, bytes, s));
    uint64_t *d_off = reinterpret_cast<uint64_t *>(buf);
    uint32_t *d_qd = reinterpret_cast<uint32_t *>(d_off + nq + 1);
    float *d_qv = reinterpret_cast<float *>(d_qd + nqp);
    cdb_status rc = CDB_OK;
    cudaError_t e = cudaMemcpyAsync(d_off, q_offsets, ((size_t)nq + 1) * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nqp) e = cudaMemcpyAsync(d_qd, q_dims, nqp * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nqp) e = cudaMemcpyAsync(d_qv, q_values, nqp * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) { set_error(std::string("cudaMemcpyAsync: ") + cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    if (!rc) rc = search_all_locked(ix, d_off, d_qd, d_qv, nq, p, r.get(), s);
    cudaFreeAsync(buf, s);
    if (rc) return rc;
    *out = r.release();
    return CDB_OK;
}

cdb_status cdb_sparse_results_offsets(const cdb_sparse_results *r, uint32_t *out_n_queries, uint64_t *out_offsets) {
    CDB_REQUIRE(r && out_n_queries, "null argument");
    *out_n_queries = (uint32_t)(r->off.size() - 1);
    if (out_offsets) std::copy(r->off.begin(), r->off.end(), out_offsets);
    return CDB_OK;
}

cdb_status cdb_sparse_results_read(const cdb_sparse_results *r, uint32_t first, uint32_t n, uint32_t *out_ids, float *out_scores) {
    CDB_REQUIRE(r, "null results");
    CDB_REQUIRE((uint64_t)first + n <= r->off.size() - 1, "read range past the results' queries");
    const uint64_t b = r->off[first], e = r->off[(size_t)first + n];
    if (b == e) return CDB_OK;
    CDB_REQUIRE(out_ids && out_scores, "null output");
    std::copy(r->ids.begin() + b, r->ids.begin() + e, out_ids);
    std::copy(r->scores.begin() + b, r->scores.begin() + e, out_scores);
    return CDB_OK;
}

cdb_status cdb_sparse_results_destroy(cdb_sparse_results *r) {
    delete r;
    return CDB_OK;
}

cdb_status cdb_sparse_sample_upper_bound(int32_t device, const float *values, uint64_t n, float clamp_margin_percent,
                                         const uint64_t *prior_counts, uint64_t prior_values, uint64_t *out_counts, float *out_ub) {
    CDB_REQUIRE((values || !n) && (out_counts || out_ub), "bad arguments");
    CDB_CUDA_TRY(cudaSetDevice(device));
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    StreamGuard sg;
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&sg.s, cudaStreamNonBlocking));
    cudaStream_t s = sg.s;
    const uint64_t chunk = 16ull << 20;
    float *d_in = nullptr;
    unsigned long long *d_c = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&d_c, 9 * 8, s));
    cdb_status rc = CDB_OK;
    cudaError_t e = cudaMemsetAsync(d_c, 0, 9 * 8, s);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_in, std::min(std::max<uint64_t>(n, 1), chunk) * 4, s);
    for (uint64_t off = 0; off < n && e == cudaSuccess; off += chunk) {
        const uint64_t m = std::min(chunk, n - off);
        e = cudaMemcpyAsync(d_in, values + off, m * 4, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) break;
        const uint32_t grid = (uint32_t)std::min<uint64_t>((m + 255) / 256, (uint64_t)sms * 8);
        sp_sample_kernel<<<grid, 256, 0, s>>>(d_in, m, d_c);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
    }
    uint64_t c[9];
    if (e == cudaSuccess) e = cudaMemcpyAsync(c, d_c, sizeof(c), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (d_in) cudaFreeAsync(d_in, s);
    cudaFreeAsync(d_c, s);
    if (e != cudaSuccess) { set_error(std::string("sparse sampling: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    for (int i = 0; i < 9; ++i) {
        if (prior_counts) c[i] += prior_counts[i];
        if (out_counts) out_counts[i] = c[i];
    }
    // finalize_sampling (inverted/mod.rs:194-247): (count as f32 / values_collected as f32) * 100.0, first t with
    // pct <= clamp_margin_percent, else 10.0 (also when no value was sampled: 0/0 is NaN)
    if (out_ub) {
        const float vc = (float)(n + (prior_counts ? prior_values : 0));
        float ub = 10.0f;
        for (int i = 0; i < 9; ++i) {
            volatile float r = (float)c[i] / vc;
            if (r * 100.0f <= clamp_margin_percent) { ub = (float)(i + 1); break; }
        }
        *out_ub = ub;
    }
    return rc;
}

}  // extern "C"
