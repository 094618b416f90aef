// kernels.h -- internal launch wrappers shared between the .cu files.
#pragma once
#include <vector>

#include "common.cuh"
#include "scorers.cuh"

namespace cdb {

// ---- quantize.cu
cdb_status quantize_rows_device(const float *d_vecs, uint64_t n, uint32_t dim, int st, float lo, float hi,
                                uint8_t *d_codes, uint32_t row_pitch, float *d_mags, float *d_raw,
                                uint32_t raw_pitch_elems, cudaStream_t s);
cdb_status quantize_rows_synth(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t dim, int st, float lo, float hi,
                               uint8_t *d_codes, uint32_t row_pitch, float *d_mags, float *d_raw,
                               uint32_t raw_pitch_elems, cudaStream_t s);
cdb_status raw_mags_device(const float *d_raw, uint32_t pitch_elems, uint64_t n, uint32_t dim, float *d_mags, cudaStream_t s);

// ---- sampling.cu
cdb_status sample_counts_device(const float *d_vecs, uint64_t n_values, unsigned long long *d_counts, int sm_count, cudaStream_t s);
void values_range_from_counts(const uint64_t *counts, uint64_t n_values, float clamp_margin_percent, float *range);

// ---- pairs.cu
cdb_status distance_pairs_device(int metric, int st, uint32_t dim, const uint8_t *d_x, const float *d_xm,
                                 const uint8_t *d_y, const float *d_ym, uint32_t row_pitch, uint64_t n,
                                 float *d_out, int32_t *d_status, cudaStream_t s);
// one side of a batch of VectorData (device pointers; nullptr = None for every element)
struct MdBatchDev {
    const uint8_t *codes;
    const float *mags;
    const uint32_t *ids;
    const uint8_t *has_id;
    const int32_t *md_bits;
    const float *md_mags;
    const uint8_t *has_md;
};
cdb_status distance_pairs_md_device(int metric, int st, uint32_t dim, uint32_t M, const MdBatchDev &x, const MdBatchDev &y,
                                    uint32_t row_pitch, uint64_t n, float *d_out, int32_t *d_status, cudaStream_t s);
// gather-score: one query against rows ids[0..n) of a stored matrix
cdb_status score_ids_device(int metric, int st, uint32_t dim, const uint8_t *d_q, float qmag,
                            const uint8_t *d_rows, const float *d_mags, uint32_t row_pitch, uint64_t n_rows,
                            const uint32_t *d_ids, uint32_t n, float *d_out, int32_t *d_status, cudaStream_t s);
// batched exact f32 cosine re-rank (finalize_ann_results): for each query b, score candidates
// cand[b*ncand .. ) (CDB_INVALID_ID = skip), write sorted top-k keys as ids/scores.
cdb_status rerank_f32_device(const float *d_raw, uint32_t pitch_elems, const float *d_raw_mags, uint64_t n_rows,
                             uint32_t dim, const float *d_q, uint32_t q_pitch_elems, const float *d_qmags, uint32_t nq,
                             const uint32_t *d_cand, const uint32_t *d_cand_counts, uint32_t ncand, uint32_t k, uint32_t id_base,
                             uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s,
                             const uint32_t *d_labels = nullptr,    // labels: ids reported instead of the candidate ids (replica ids)
                             uint64_t *d_out_keys = nullptr);       // [nq][k] packed selection keys as well (shard merge)

// ---- scan.cu
struct ScanArgs {
    const uint8_t *rows;   // stored matrix (codes or raw f32), row-pitched
    uint32_t row_pitch;    // bytes
    const float *mags;     // per-row magnitude used by the formula
    uint64_t n;
    uint32_t dim;
    int st;                // storage type of `rows`
    int metric;
    int raw_mode;          // 1: finalize formula (no zero check), 0: DistanceMetric::calculate
    const uint8_t *q;      // prepared queries, same layout/pitch as rows
    const float *qmags;
    uint32_t nq;
    uint32_t k;
    uint32_t id_base;
    uint64_t *partial;     // [nq][nsplit][k] selection keys
    uint32_t nsplit;
    uint32_t *err32;       // [nq] error bits (atomicOr) or null
    // Device-side fallback decision of the tensor-core paths (no host sync).  qsel = {n_sel, query indices...} is written by
    // select_fallback_kernel.  Two launches share it:
    //   selective (sel_mode = 1): 1-D grid; runs only if 0 < n_sel <= sel_cap, over the selected queries only -- the CTAs
    //       split themselves over ceil(n_sel/QB) query groups, so a single bad query gets the whole GPU;
    //   full      (sel_mode = 0): the whole batch, runs only if qsel == null (no tensor path) or n_sel > sel_cap.
    const uint32_t *qsel;
    uint32_t sel_cap;
    int sel_mode;
    uint32_t sel_grid;   // CTAs of the selective launch (scan_sel_grid)
};
constexpr uint32_t SCAN_SEL_CAP = 64;
// picks grid/template; returns nsplit chosen through args.nsplit (caller sizes `partial` with scan_max_partials)
uint32_t scan_plan_nsplit(const ScanArgs &a, int sm_count);
cdb_status scan_topk_device(const ScanArgs &a, cudaStream_t s);
// partial [nq][nsplit][k] -> ids/scores/counts
cdb_status merge_partials_device(int metric, const uint64_t *d_partial, uint32_t nq, uint32_t nlists, uint32_t k,
                                 uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t s,
                                 const uint32_t *qsel = nullptr, uint32_t sel_cap = 0, int sel_mode = 0, uint32_t sel_grid = 0, uint32_t sel_qb = 0,
                                 uint64_t *d_out_keys = nullptr);
// grid of the selective scan (CTAs) and its query block; the partial buffer needs SCAN_SEL_CAP * grid * k keys
uint32_t scan_sel_grid(int sm_count, uint32_t k);
uint32_t scan_sel_qb(const ScanArgs &a);
// [n_shards][nq][k] ids/scores -> keys [nq][n_shards][k]
cdb_status pack_keys_device(int metric, const uint32_t *d_ids, const float *d_scores, uint32_t n_shards, uint32_t nq,
                            uint32_t k, uint64_t *d_keys, cudaStream_t s);

// ---- hnsw.cu
struct GraphDev {
    uint32_t num_levels, nbrs, nbrs0, entry, root_row;
    uint32_t identity_mask;           // bit L: node_row[L][i] == i for every node of level L (the lookup is skipped)
    const uint32_t *const *node_row;  // device arrays of device pointers, [num_levels+1]
    const uint32_t *const *adj;
    const uint32_t *const *child;
};
struct HnswArgs {
    GraphDev g;
    const uint8_t *rows;
    uint32_t row_pitch;
    const float *mags;
    uint32_t dim;
    int st, metric;
    const uint8_t *q;
    const float *qmags;
    uint32_t nq, ef, shortlist;
    uint32_t out_cap;
    uint32_t *out_rows;
    float *out_scores;
    uint32_t *out_n;
    uint32_t *err32;
    unsigned long long *counters;
    unsigned long long *prof;         // null, or clock64 sums (hnsw_warp.cu)
    uint32_t flags;                   // CDB_HNSW_F_* variant switches of the warp kernel
};
// variant switches of hnsw_search_warp_kernel (cdb_debug_set_hnsw_flags; the default is the best measured combination)
constexpr uint32_t CDB_HNSW_F_PRELOAD = 2;   // load the next head's adjacency slots while the queue merge runs
constexpr uint32_t CDB_HNSW_F_ATOMFS = 4;    // fixed-set walk through atomicOr return values (slot-order loop only on aliasing)
constexpr uint32_t CDB_HNSW_F_CTA = 8;       // round-1 kernel: one CTA per query
constexpr uint32_t CDB_HNSW_F_SPEC = 32;     // idle lanes of a chain phase score the next heads' neighbours ahead of time (hnsw_warp.cu)
constexpr uint32_t CDB_HNSW_F_POOL = 16;     // candidates as an unsorted pool + arg-max pops instead of a sorted queue + merges
constexpr uint32_t CDB_HNSW_F_DEFAULT = CDB_HNSW_F_PRELOAD | CDB_HNSW_F_ATOMFS;
extern std::atomic<uint32_t> g_hnsw_flags;
cdb_status hnsw_search_device(const HnswArgs &a, cudaStream_t s);        // one CTA per query (round-1 kernel; A/B runs)
cdb_status hnsw_search_warp_device(const HnswArgs &a, cudaStream_t s);   // one warp per query (hnsw_warp.cu)
cdb_status hnsw_dedup_device(const uint32_t *d_rows, const float *d_scores, const uint32_t *d_n, uint32_t in_cap, int metric,
                             uint32_t root_row, uint32_t id_base, uint32_t k5, uint32_t nq, uint32_t *d_cand, uint32_t *d_cand_cnt,
                             cudaStream_t s);

// ---- hnsw_md.cu (metadata-filtered search on graphs with replica nodes)
struct HnswMdArgs {
    HnswArgs a;                       // out_rows = vector row of each result (CDB_INVALID_ID for pseudo nodes)
    const uint32_t *const *node_id;   // device table [num_levels+1] of device arrays
    const uint32_t *const *node_md;
    const int32_t *md_bits;           // [n_md][M]
    const float *md_mags;
    uint32_t M;
    uint32_t pseudo_entry;
    const uint32_t *filter_offsets;   // [nq+1] rows of filter_dims per query
    const int8_t *filter_dims;        // [total][M]
    const uint8_t *has_filter;        // [nq] (nullptr = no query has a filter)
    uint32_t *out_ids;                // [nq][out_cap] replica ids
};
cdb_status hnsw_search_md_device(const HnswMdArgs &a, cudaStream_t s);
cdb_status hnsw_dedup_md_device(const uint32_t *d_ids, const uint32_t *d_rows, const float *d_scores, const uint32_t *d_n,
                                uint32_t in_cap, int metric, uint32_t id_base, uint32_t k5, uint32_t nq, uint32_t *d_cand,
                                uint32_t *d_labels, uint32_t *d_cand_cnt, cudaStream_t s);

// ---- hnsw_build.cu
struct HnScoreCtx;
cdb_status hnsw_build_device(const HnScoreCtx &sc, uint32_t n, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0,
                             uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t seed, GraphDev *out_graph,
                             std::vector<void *> *out_allocs, std::vector<uint32_t> *out_counts,
                             std::vector<const uint32_t *> *out_nr, std::vector<const uint32_t *> *out_ad,
                             std::vector<const uint32_t *> *out_ch, cudaStream_t s);

// replica lists: one entry per graph node to create, host arrays (cdb_replica_build)
struct ReplicaHost {
    uint32_t n_nodes;
    const uint32_t *row, *node_id, *base_id, *md_row;
    const uint8_t *max_level;
    uint32_t md_dims, n_md;
    const int32_t *md_bits;
    const float *md_mags;
    uint32_t main_root_row, main_root_md, pseudo_root_row, pseudo_root_md;
};
struct ReplicaGraphDev {
    const uint32_t *const *node_id, *const *node_md;   // device tables of device arrays
    std::vector<const uint32_t *> h_node_id, h_node_md;   // the same per-level device pointers on the host
    const int32_t *md_bits;
    const float *md_mags;
    uint32_t md_dims, pseudo_entry;
};
cdb_status hnsw_build_replicas_device(const HnScoreCtx &sc, const ReplicaHost &rh, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0,
                                      uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, GraphDev *out_graph,
                                      std::vector<void *> *out_allocs, std::vector<uint32_t> *out_counts,
                                      std::vector<const uint32_t *> *out_nr, std::vector<const uint32_t *> *out_ad,
                                      std::vector<const uint32_t *> *out_ch, ReplicaGraphDev *out_md, std::vector<uint8_t> *out_failed,
                                      cudaStream_t s);

// ---- tensor_scan.cu (wgmma prefilter)
constexpr uint32_t TS_MAX_ODD = 64;   // degenerate rows that are not all-zero ride on every candidate list; more -> no prefilter
constexpr uint32_t TS_DEG_WORDS = 2 + TS_MAX_ODD;
cdb_status normalize_f16_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t n, uint32_t dim,
                                void *d_out, uint32_t out_pitch_halfs, cudaStream_t s);
cdb_status classify_rows_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t n, uint32_t dim,
                                uint32_t first_row, uint32_t *d_deg, cudaStream_t s);
size_t tensor_scan_smem_bytes(uint32_t k);
cdb_status tensor_scan_device(const void *d_xh, const void *d_qh, uint32_t pitch_halfs, uint64_t n_rows, uint32_t nq,
                              uint32_t dim, uint32_t k, float two_eps, uint32_t id_base, int *d_ggm, uint32_t *d_cand,
                              uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_progress /* 2048 words */, const uint32_t *d_deg,
                              bool has_deg, int sm_count, cudaStream_t s, bool prepared = false);
// one launch: raw + fp16-normalised query copies, |q|, and every per-search initialisation of the prefilter path
cdb_status prep_queries_device(const float *d_q, uint32_t nq, uint32_t dim, float *d_q_raw, uint32_t raw_pitch_elems, float *d_q_mags,
                               void *d_qh, uint32_t qh_pitch_halfs, int *d_ggm, const uint32_t *d_deg, bool has_deg, uint32_t id_base,
                               uint32_t *d_cand, uint32_t cand_cap, uint32_t *d_cand_cnt, uint32_t *d_err32, uint8_t *d_err8,
                               uint32_t *d_progress, cudaStream_t s);
cdb_status tensor_scan_i8_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_ggm,
                                 uint64_t *d_cand64, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32,
                                 uint32_t *d_progress /* 2048 words */, int sm_count, cudaStream_t s);
// queries whose candidate list overflowed (or whose norm is degenerate, d_qmags may be null) -> d_qsel = {n, indices...}
cdb_status select_fallback_device(const uint32_t *d_cnt, uint32_t cap, const float *d_qmags, uint32_t n, uint32_t *d_qsel,
                                  uint32_t *d_flags, cudaStream_t s);

// ---- tensor_scan_u8.cu (exact integer scoring on wgmma u8)
size_t tensor_u8_smem_bytes(uint32_t k);
cdb_status unpack_digits_device(const uint8_t *d_codes, uint32_t row_pitch, uint64_t n, uint32_t dim, int res, uint8_t *d_out,
                                uint32_t out_pitch, cudaStream_t s);
cdb_status tensor_u8_scan_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_gthr,
                                 uint64_t *d_cand, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32, uint32_t *d_progress,
                                 uint32_t *d_ids, float *d_scores, uint32_t *d_counts, int sm_count, cudaStream_t s,
                                 uint64_t *d_out_keys = nullptr);

}  // namespace cdb
