// hnsw.cu -- the step between the HNSW traversal (hnsw_warp.cu) and the exact re-rank (S1, CDB_MODE_HNSW):
//   remove_duplicates_and_filter  src/models/common.rs:381-412
//   get_raw_emb_by_internal_id    src/models/collection.rs:368-384 (replica id -> base vector: the result's row)
#include "hnsw_traverse.cuh"

namespace cdb {

// remove_duplicates_and_filter: dedup by id keeping the first occurrence, drop the root, sort best-first, truncate to 5*k.
// One CTA per query; writes global candidate ids (id_base + row) for the re-rank.  The id of an entry is ids[i] (replica ids
// on graphs with metadata) or, with ids == null, its row.  Dropped: id == drop_id (the root: its row on plain graphs,
// u32::MAX on replica graphs) and pseudo nodes (row == CDB_INVALID_ID).  labels (may be null) = the kept entries' ids.
__global__ void __launch_bounds__(256) hnsw_dedup_kernel(const uint32_t *__restrict__ ids, const uint32_t *__restrict__ rows,
                                                         const float *__restrict__ scores, const uint32_t *__restrict__ n_in,
                                                         uint32_t in_cap, int metric, uint32_t drop_id, uint32_t id_base, uint32_t k5,
                                                         uint32_t *__restrict__ cand, uint32_t *__restrict__ labels,
                                                         uint32_t *__restrict__ cand_cnt) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    uint32_t P = 1;
    while (P < in_cap) P <<= 1;
    uint32_t *vals = reinterpret_cast<uint32_t *>(keys + P);   // source position of the entry
    uint32_t *sid = vals + P;
    __shared__ int kept;
    const uint32_t q = blockIdx.x, n = min(n_in[q], in_cap);
    const uint32_t *qids = (ids ? ids : rows) + (size_t)q * in_cap, *qrows = rows + (size_t)q * in_cap;
    if (threadIdx.x == 0) kept = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) sid[i] = qids[i];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t id = sid[i];
        bool dup = false;
        for (uint32_t j = 0; j < i; ++j) dup |= sid[j] == id;
        uint64_t key = 0;
        if (!dup && id != drop_id && qrows[i] != CDB_INVALID_ID) {
            key = make_key64(order_key(metric, __float_as_uint(scores[(size_t)q * in_cap + i])), id);
            atomicAdd(&kept, 1);
        }
        keys[i] = key;
        vals[i] = i;
    }
    __syncthreads();
    // sort descending (0 = dropped entries last; the kept keys are distinct: their ids are)
    for (uint32_t i = n + threadIdx.x; i < P; i += blockDim.x) { keys[i] = 0ull; vals[i] = 0; }
    __syncthreads();
    for (uint32_t size = 2; size <= P; size <<= 1)
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) { keys[lo] = y; keys[hi] = x; const uint32_t v = vals[lo]; vals[lo] = vals[hi]; vals[hi] = v; }
            }
            __syncthreads();
        }
    const uint32_t m = min((uint32_t)kept, k5);
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        cand[(size_t)q * k5 + i] = id_base + qrows[vals[i]];
        if (labels) labels[(size_t)q * k5 + i] = sid[vals[i]];
    }
    if (threadIdx.x == 0) cand_cnt[q] = m;
}

cdb_status hnsw_dedup_device(const uint32_t *d_ids, const uint32_t *d_rows, const float *d_scores, const uint32_t *d_n, uint32_t in_cap,
                             int metric, uint32_t drop_id, uint32_t id_base, uint32_t k5, uint32_t nq, uint32_t *d_cand,
                             uint32_t *d_labels, uint32_t *d_cand_cnt, cudaStream_t s) {
    if (!nq) return CDB_OK;
    uint32_t P = 1;
    while (P < in_cap) P <<= 1;
    const size_t smem = (size_t)P * 12 + (size_t)in_cap * 4 + 16;
    if (smem > 200 * 1024) { set_error("hnsw dedup: too many levels"); return CDB_INVALID_PARAMS; }
    CDB_ALLOW_SMEM(hnsw_dedup_kernel, smem);
    hnsw_dedup_kernel<<<nq, 256, smem, s>>>(d_ids, d_rows, d_scores, d_n, in_cap, metric, drop_id, id_base, k5, d_cand, d_labels,
                                            d_cand_cnt);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
