// pairs.cu -- pairwise DistanceFunction::calculate (src/models/types.rs:469-495),
// gather-score for neighbour expansion (S2, src/vector_store.rs:1161-1191) and the
// exact f32 re-rank of finalize_ann_results (S3, src/vector_store.rs:404-445).
#include "kernels.h"
#include "metadata.cuh"

namespace cdb {

__global__ void distance_pairs_kernel(int metric, int st, uint32_t dim, const uint8_t *__restrict__ x,
                                      const float *__restrict__ xm, const uint8_t *__restrict__ y,
                                      const float *__restrict__ ym, uint32_t pitch, uint64_t n,
                                      float *__restrict__ out, int32_t *__restrict__ status) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t pp = plane_pitch(dim);
    float v = 0.0f;
    int rc = pair_distance(metric, st, dim, x + i * pitch, xm[i], pp, y + i * pitch, ym[i], pp, &v);
    out[i] = rc == CDB_OK ? v : 0.0f;
    status[i] = rc;
}

cdb_status distance_pairs_device(int metric, int st, uint32_t dim, const uint8_t *d_x, const float *d_xm,
                                 const uint8_t *d_y, const float *d_ym, uint32_t row_pitch, uint64_t n,
                                 float *d_out, int32_t *d_status, cudaStream_t s) {
    if (!n) return CDB_OK;
    distance_pairs_kernel<<<(uint32_t)((n + 63) / 64), 64, 0, s>>>(metric, st, dim, d_x, d_xm, d_y, d_ym, row_pitch, n, d_out, d_status);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// DistanceMetric::calculate with metadata (replica-kind arms, cosine.rs:34-102); one thread per pair
__global__ void distance_pairs_md_kernel(int metric, int st, uint32_t dim, uint32_t M, MdBatchDev x, MdBatchDev y, uint32_t pitch,
                                         uint64_t n, float *__restrict__ out, int32_t *__restrict__ status) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t pp = plane_pitch(dim);
    auto side = [&](const MdBatchDev &b) {
        const bool has_md = b.md_bits && (!b.has_md || b.has_md[i]);
        return MdSide{b.codes + i * pitch, b.mags[i], pp, b.ids && (!b.has_id || b.has_id[i]), b.ids ? b.ids[i] : 0u,
                      has_md ? b.md_bits + i * M : nullptr, has_md ? b.md_mags[i] : 0.0f};
    };
    float v = 0.0f;
    const int rc = md_pair_distance(metric, st, dim, M, side(x), side(y), &v);
    out[i] = rc == CDB_OK ? v : 0.0f;
    status[i] = rc;
}

cdb_status distance_pairs_md_device(int metric, int st, uint32_t dim, uint32_t M, const MdBatchDev &x, const MdBatchDev &y,
                                    uint32_t row_pitch, uint64_t n, float *d_out, int32_t *d_status, cudaStream_t s) {
    if (!n) return CDB_OK;
    distance_pairs_md_kernel<<<(uint32_t)((n + 63) / 64), 64, 0, s>>>(metric, st, dim, M, x, y, row_pitch, n, d_out, d_status);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// one thread per id; the query row sits in global memory (L1/L2 resident)
__global__ void score_ids_kernel(int metric, int st, uint32_t dim, const uint8_t *__restrict__ q, float qmag,
                                 const uint8_t *__restrict__ rows, const float *__restrict__ mags, uint32_t pitch,
                                 uint64_t n_rows, const uint32_t *__restrict__ ids, uint32_t n,
                                 float *__restrict__ out, int32_t *__restrict__ status) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = ids[i];
    if (id >= n_rows) { out[i] = 0.0f; status[i] = CDB_INVALID_PARAMS; return; }
    const uint32_t pp = plane_pitch(dim);
    float v = 0.0f;
    int rc = pair_distance(metric, st, dim, q, qmag, pp, rows + (size_t)id * pitch, mags[id], pp, &v);
    out[i] = rc == CDB_OK ? v : 0.0f;
    status[i] = rc;
}

cdb_status score_ids_device(int metric, int st, uint32_t dim, const uint8_t *d_q, float qmag,
                            const uint8_t *d_rows, const float *d_mags, uint32_t row_pitch, uint64_t n_rows,
                            const uint32_t *d_ids, uint32_t n, float *d_out, int32_t *d_status, cudaStream_t s) {
    if (!n) return CDB_OK;
    score_ids_kernel<<<(n + 63) / 64, 64, 0, s>>>(metric, st, dim, d_q, qmag, d_rows, d_mags, row_pitch, n_rows, d_ids, n, d_out, d_status);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// ------------------------------------------------------------------ exact re-rank
// One CTA per query.  Eight consecutive lanes score one candidate: lane j owns AVX
// lane j of dot_product_f32_simd, so a group reads 32 contiguous bytes per step and
// the xor-butterfly reproduces the reference's hadd tree.  cs = dp / (|q|*|v|) with
// no zero check (vector_store.rs:427-429); sort by total_cmp desc, truncate k.
// The candidate list is consumed in chunks through a fixed 2048-key buffer (best keys of the earlier chunks stay at
// the front), so shared memory does not grow with the list and long prefilter lists cost time, not occupancy.
// With `dedup`, a candidate id may appear twice (degenerate rows are pre-seeded on prefilter lists and may be emitted
// again): equal keys are adjacent after the sort and are reported once -- at most RERANK_DUP of them, which bounds the
// copies a prefilter list can hold.  Without it every candidate is reported, copies included, as finalize_ann_results
// reports them.
constexpr int RERANK_THREADS = 256;
constexpr uint32_t RERANK_BUF = 2048;
constexpr uint32_t RERANK_DUP = 64;    // duplicates tolerated inside the kept window

__device__ inline void rerank_sort_desc(uint64_t *keys, uint32_t n) {
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = n + threadIdx.x; i < P; i += blockDim.x) keys[i] = 0ull;
    __syncthreads();
    for (uint32_t size = 2; size <= P; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1));  // index with bit `stride` clear
                const uint32_t hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) { keys[lo] = y; keys[hi] = x; }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(RERANK_THREADS) rerank_f32_kernel(
    const float *__restrict__ raw, uint32_t pitch_elems, const float *__restrict__ raw_mags, uint64_t n_rows,
    uint32_t dim, const float *__restrict__ q, uint32_t q_pitch_elems, const float *__restrict__ qmags,
    const uint32_t *__restrict__ cand, const uint32_t *__restrict__ cand_counts, uint32_t cand_stride, uint32_t k, uint32_t id_base,
    uint32_t *__restrict__ out_ids, float *__restrict__ out_scores, uint32_t *__restrict__ out_counts,
    const uint32_t *__restrict__ labels, uint64_t *__restrict__ out_keys, const uint32_t *__restrict__ deleted, bool dedup) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *qs = reinterpret_cast<float *>(smem);
    uint64_t *keys = reinterpret_cast<uint64_t *>(qs + round_up(dim, 4));
    __shared__ int nvalid;
    __shared__ uint32_t ndup, duppos[RERANK_DUP];
    const uint32_t b = blockIdx.x;
    const uint32_t ncand = cand_counts ? min(cand_counts[b], cand_stride) : cand_stride;
    for (uint32_t c = threadIdx.x; c < dim; c += blockDim.x) qs[c] = q[(size_t)b * q_pitch_elems + c];
    for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) {
        out_ids[(size_t)b * k + j] = CDB_INVALID_ID;
        out_scores[(size_t)b * k + j] = 0.0f;
        if (out_keys) out_keys[(size_t)b * k + j] = 0ull;   // packed selection keys for the shard merge (0 = empty slot)
    }
    if (threadIdx.x == 0) { nvalid = 0; ndup = 0; }
    __syncthreads();
    const float mag_q = qmags[b];
    const int j = threadIdx.x & 7, grp = threadIdx.x >> 3;
    const uint32_t window = min(k + RERANK_DUP, RERANK_BUF / 2);   // keys carried from chunk to chunk
    uint32_t kept = 0, pos = 0, n = 0;
    do {
        const uint32_t take = min(RERANK_BUF - kept, ncand - pos);
        const uint32_t rounds = (take + RERANK_THREADS / 8 - 1) / (RERANK_THREADS / 8);
        for (uint32_t r = 0; r < rounds; ++r) {
            const uint32_t ci = r * (RERANK_THREADS / 8) + grp;   // within this chunk
            uint32_t id = ci < take ? cand[(size_t)b * cand_stride + pos + ci] : CDB_INVALID_ID;
            // deleted rows reach the list through a zero shadow row emitted at a threshold <= 0, or as pre-seeded odd rows
            bool ok = id != CDB_INVALID_ID && id >= id_base && (uint64_t)(id - id_base) < n_rows;
            if (ok && deleted) ok = !((deleted[(id - id_base) >> 5] >> ((id - id_base) & 31)) & 1u);
            const uint64_t rowi = ok ? (uint64_t)(id - id_base) : 0;
            float dp = dot_f32_avx_order_8t(qs, raw + rowi * pitch_elems, dim, j);  // all lanes participate in the shuffles
            if (j == 0 && ci < take) {
                uint64_t key = 0;
                if (ok) {
                    float cs = canon_nan(__fdiv_rn(dp, __fmul_rn(mag_q, raw_mags[rowi])));
                    key = make_key64(order_key(CDB_METRIC_COSINE, __float_as_uint(cs)), labels ? labels[(size_t)b * cand_stride + pos + ci] : id);
                }
                keys[kept + ci] = key;
                if (ok) atomicAdd(&nvalid, 1);
            }
        }
        __syncthreads();
        n = kept + take;
        rerank_sort_desc(keys, n);   // zero (empty) keys sort last
        pos += take;
        kept = min(n, window);
    } while (pos < ncand);
    // equal keys (same score, same id) are duplicates of one candidate: report the first of each run
    const uint32_t lim = min(n, window);
    for (uint32_t i = 1 + threadIdx.x; dedup && i < lim; i += blockDim.x)
        if (keys[i] != 0ull && keys[i] == keys[i - 1]) {
            const uint32_t p = atomicAdd(&ndup, 1u);
            if (p < RERANK_DUP) duppos[p] = i;
        }
    __syncthreads();
    const uint32_t nd = min(ndup, RERANK_DUP);
    const uint32_t have = min((uint32_t)nvalid, lim);            // non-empty keys inside the window
    const uint32_t uniq = have > nd ? have - nd : 0;
    const uint32_t nout = uniq < k ? uniq : k;
    for (uint32_t i = threadIdx.x; i < have; i += blockDim.x) {
        const uint64_t key = keys[i];
        uint32_t shift = 0;
        bool dup = false;
        for (uint32_t d = 0; d < nd; ++d) { shift += duppos[d] < i; dup |= duppos[d] == i; }
        const uint32_t o = i - shift;
        if (!dup && o < nout) {
            out_ids[(size_t)b * k + o] = key64_id(key);
            out_scores[(size_t)b * k + o] = __uint_as_float(key_to_bits(CDB_METRIC_COSINE, (uint32_t)(key >> 32)));
            if (out_keys) out_keys[(size_t)b * k + o] = key;
        }
    }
    if (threadIdx.x == 0 && out_counts) out_counts[b] = nout;
}

uint32_t rerank_f32_max_dim() { return (200 * 1024 - RERANK_BUF * 8) / 4; }

cdb_status rerank_f32_device(const float *d_raw, uint32_t pitch_elems, const float *d_raw_mags, uint64_t n_rows,
                             uint32_t dim, const float *d_q, uint32_t q_pitch_elems, const float *d_qmags, uint32_t nq,
                             const uint32_t *d_cand, const uint32_t *d_cand_counts, uint32_t ncand, uint32_t k, uint32_t id_base,
                             uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s,
                             const uint32_t *d_labels, uint64_t *d_out_keys, const uint32_t *d_deleted, bool dedup) {
    if (!nq) return CDB_OK;
    if (k == 0 || k > 1024) { set_error("rerank: k must be in 1..1024"); return CDB_INVALID_PARAMS; }
    uint32_t pcap = 64;
    while (pcap < ncand && pcap < RERANK_BUF) pcap <<= 1;
    if (ncand > pcap) pcap = RERANK_BUF;
    size_t smem = (size_t)round_up(dim, 4) * 4 + (size_t)pcap * 8;
    if (smem > 200 * 1024) { set_error("rerank: dimension too large"); return CDB_INVALID_PARAMS; }
    CDB_ALLOW_SMEM(rerank_f32_kernel, smem);
    rerank_f32_kernel<<<nq, RERANK_THREADS, smem, s>>>(d_raw, pitch_elems, d_raw_mags, n_rows, dim, d_q, q_pitch_elems,
                                                        d_qmags, d_cand, d_cand_counts, ncand, k, id_base, d_out_ids, d_out_scores, d_out_counts, d_labels, d_out_keys,
                                                        d_deleted, dedup);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// finalize_ann_results with top_k None: every candidate of the query is scored and the whole list is sorted and returned
// (vector_store.rs:404-445 without the truncation).  One CTA per query holds all of its keys at once, so the list is bounded
// by the HNSW output, (num_levels + 1) * 100 <= 3200 candidates; the arithmetic, the key and the order are those of
// rerank_f32_kernel.  The candidates' keys are unique (hnsw_dedup_kernel removed repeated ids), so nothing is deduplicated.
// Row q of the outputs has `width` columns: the counts[q] sorted results, then CDB_INVALID_ID / 0 (keys 0).
constexpr int RERANK_ALL_THREADS = 512;

__global__ void __launch_bounds__(RERANK_ALL_THREADS) rerank_all_f32_kernel(
    const float *__restrict__ raw, uint32_t pitch_elems, const float *__restrict__ raw_mags, uint64_t n_rows,
    uint32_t dim, const float *__restrict__ q, uint32_t q_pitch_elems, const float *__restrict__ qmags,
    const uint32_t *__restrict__ cand, const uint32_t *__restrict__ cand_counts, uint32_t cand_stride, uint32_t width,
    uint32_t id_base, uint32_t *__restrict__ out_ids, float *__restrict__ out_scores, uint32_t *__restrict__ out_counts,
    const uint32_t *__restrict__ labels, uint64_t *__restrict__ out_keys) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *qs = reinterpret_cast<float *>(smem);
    uint64_t *keys = reinterpret_cast<uint64_t *>(qs + round_up(dim, 4));
    __shared__ int nvalid;
    const uint32_t b = blockIdx.x;
    const uint32_t ncand = min(cand_counts[b], cand_stride);
    for (uint32_t c = threadIdx.x; c < dim; c += blockDim.x) qs[c] = q[(size_t)b * q_pitch_elems + c];
    if (threadIdx.x == 0) nvalid = 0;
    __syncthreads();
    const float mag_q = qmags[b];
    const int j = threadIdx.x & 7, grp = threadIdx.x >> 3;
    const uint32_t rounds = (ncand + RERANK_ALL_THREADS / 8 - 1) / (RERANK_ALL_THREADS / 8);
    for (uint32_t r = 0; r < rounds; ++r) {
        const uint32_t ci = r * (RERANK_ALL_THREADS / 8) + grp;
        const uint32_t id = ci < ncand ? cand[(size_t)b * cand_stride + ci] : CDB_INVALID_ID;
        const bool ok = id != CDB_INVALID_ID && id >= id_base && (uint64_t)(id - id_base) < n_rows;
        const uint64_t rowi = ok ? (uint64_t)(id - id_base) : 0;
        const float dp = dot_f32_avx_order_8t(qs, raw + rowi * pitch_elems, dim, j);   // all lanes take part in the shuffles
        if (j == 0 && ci < ncand) {
            uint64_t key = 0;
            if (ok) {
                const float cs = canon_nan(__fdiv_rn(dp, __fmul_rn(mag_q, raw_mags[rowi])));
                key = make_key64(order_key(CDB_METRIC_COSINE, __float_as_uint(cs)), labels ? labels[(size_t)b * cand_stride + ci] : id);
                atomicAdd(&nvalid, 1);
            }
            keys[ci] = key;
        }
    }
    __syncthreads();
    rerank_sort_desc(keys, ncand);   // zero (empty) keys sort last
    const uint32_t nout = min((uint32_t)nvalid, width);
    for (uint32_t i = threadIdx.x; i < width; i += blockDim.x) {
        const uint64_t key = i < nout ? keys[i] : 0ull;
        out_ids[(size_t)b * width + i] = key ? key64_id(key) : CDB_INVALID_ID;
        out_scores[(size_t)b * width + i] = key ? __uint_as_float(key_to_bits(CDB_METRIC_COSINE, (uint32_t)(key >> 32))) : 0.0f;
        if (out_keys) out_keys[(size_t)b * width + i] = key;
    }
    if (threadIdx.x == 0 && out_counts) out_counts[b] = nout;
}

bool rerank_all_fits(uint32_t dim, uint32_t ncand) {
    uint32_t P = 1;
    while (P < ncand) P <<= 1;
    return ncand <= RERANK_ALL_MAX_CAND && (size_t)round_up(dim, 4) * 4 + (size_t)P * 8 <= 200 * 1024;
}

cdb_status rerank_all_f32_device(const float *d_raw, uint32_t pitch_elems, const float *d_raw_mags, uint64_t n_rows, uint32_t dim,
                                 const float *d_q, uint32_t q_pitch_elems, const float *d_qmags, uint32_t nq, const uint32_t *d_cand,
                                 const uint32_t *d_cand_counts, uint32_t ncand, uint32_t width, uint32_t id_base, uint32_t *d_out_ids,
                                 float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s, const uint32_t *d_labels,
                                 uint64_t *d_out_keys) {
    if (!nq) return CDB_OK;
    if (ncand == 0 || ncand > RERANK_ALL_MAX_CAND) { set_error("rerank: 1..4096 candidate slots per query"); return CDB_INVALID_PARAMS; }
    if (!rerank_all_fits(dim, ncand)) { set_error("rerank: dimension too large"); return CDB_INVALID_PARAMS; }
    uint32_t P = 1;
    while (P < ncand) P <<= 1;
    const size_t smem = (size_t)round_up(dim, 4) * 4 + (size_t)P * 8;
    CDB_ALLOW_SMEM(rerank_all_f32_kernel, smem);
    rerank_all_f32_kernel<<<nq, RERANK_ALL_THREADS, smem, s>>>(d_raw, pitch_elems, d_raw_mags, n_rows, dim, d_q, q_pitch_elems, d_qmags,
                                                               d_cand, d_cand_counts, ncand, width, id_base, d_out_ids, d_out_scores,
                                                               d_out_counts, d_labels, d_out_keys);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
