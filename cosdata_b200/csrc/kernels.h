// kernels.h -- internal launch wrappers shared between the .cu files.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "scorers.cuh"

namespace cdb {

// k of a dense search: 1..1024, or under CDB_SEARCH_ALL_CANDIDATES (top_k None, HNSW only) the output row width, which is
// checked against the graph once the handle is locked
inline cdb_status check_search_k(const cdb_search_params *p) {
    if (p->flags & CDB_SEARCH_ALL_CANDIDATES) {
        CDB_REQUIRE(p->mode == CDB_MODE_HNSW, "CDB_SEARCH_ALL_CANDIDATES (top_k None) applies to CDB_MODE_HNSW");
        return CDB_OK;
    }
    CDB_REQUIRE(p->k >= 1 && p->k <= 1024, "k must be in 1..1024");
    return CDB_OK;
}

// metadata filters of a batch in device memory, the arguments of cdb_search_batch_filtered_device (a shard group's filtered search)
struct ShardFilters {
    const uint32_t *off;   // [n_queries + 1], may be null when has is
    const int8_t *dims;    // [n_rows][md_dims]
    uint32_t n_rows;
    const uint8_t *has;    // [n_queries], null: no query has a filter
};

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

// ---- sparse.cu
// rows held, rows and pairs that still fit
cdb_status sparse_index_room(cdb_sparse_index *ix, uint64_t *rows, uint64_t *rows_left, uint64_t *pairs_left);
// drops the rows from `rows` on (their tombstones too): an append of several calls undone after a later call failed
cdb_status sparse_index_truncate(cdb_sparse_index *ix, uint64_t rows);
int sparse_index_device(const cdb_sparse_index *ix);
// The device half of a top_k None search (a single index's, and each shard's of a shard group).  One chunk of queries is
// scored, its candidates gathered per query, sorted descending and, with rerank, re-ranked and sorted again: query qi's
// keys are keys[seg_h[qi], seg_h[qi + 1]), contiguous in device memory.  The caller holds the index's reader lock.
struct SparseAllScratch {
    uint64_t *slots = nullptr, *ka = nullptr, *kb = nullptr;
    uint32_t *cnt = nullptr, *pos = nullptr, *seg = nullptr, *qa = nullptr, *qb = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    uint32_t chunk = 0;
    std::vector<uint32_t> seg_h;        // [chunk + 1], host
    const uint64_t *keys = nullptr;     // the sorted keys of the last chunk (null without candidates)
    uint64_t *spare = nullptr;          // a free buffer of as many keys
};
// tiles, and live rows (a query's candidates, at most)
void sparse_index_all_bounds(const cdb_sparse_index *ix, uint64_t *n_tiles, uint64_t *n_live);
// queries per chunk: the scratch of a chunk over at most n_tiles tiles and n_live live rows stays within 512 MB
uint32_t sparse_all_chunk(uint32_t nq, uint64_t n_tiles, uint64_t n_live);
cdb_status sparse_all_alloc(cdb_sparse_index *ix, uint32_t chunk, SparseAllScratch *sc, cudaStream_t s);
cdb_status sparse_all_keys(cdb_sparse_index *ix, const uint64_t *d_qoff, const uint32_t *d_qdims, const float *d_qvals,
                           const cdb_sparse_search_params *p, uint32_t q0, uint32_t c, SparseAllScratch *sc, cudaStream_t s);
void sparse_all_free(SparseAllScratch *sc, cudaStream_t s);

// ---- tfidf.cu
int tfidf_index_device(const cdb_tfidf_index *ix);

// ---- api.cu
int index_device(const cdb_index *ix);
uint32_t index_dim(const cdb_index *ix);
// graph metadata attached (results carry replica ids); read under the handle's shared lock
bool index_has_graph_metadata(cdb_index *ix);

// ---- hybrid.cu: the fusion of two ranked lists per query (cdb_rrf_fuse's kernel), and the request check, chunks and
// fusion of a hybrid batch, shared with the shard group's hybrid search
constexpr uint32_t HYB_MAX_TOP_K = 341;   // 3 * top_k <= 1024, the dense and sparse searches' k limit
enum HybSource { HYB_DENSE = 0, HYB_SPARSE = 1, HYB_TFIDF = 2 };
// columns of a source's intermediate list: 3 * top_k, TF-IDF at most its 512 buckets
inline uint32_t hyb_list_ld(int src, uint32_t top_k) { return std::min(3 * top_k, src == HYB_TFIDF ? 512u : 3 * top_k); }
struct RrfList {
    const uint32_t *ids;      // [B][ld]
    const uint32_t *counts;   // [B]
    uint32_t ld, stride;
    const uint32_t *rows = nullptr;   // device, [n]: the list row fused into row i (null: row i)
};
// where a fusion writes: fused row i lands in output row rows[i] (null: row i); with err, err[rows[i]] = err_in[first
// list's row] (null err_in: 0)
struct RrfRows {
    const uint32_t *rows = nullptr;
    const uint8_t *err_in = nullptr;
    uint8_t *err = nullptr;
};
cdb_status fuse_launch(const RrfList &a, const RrfList &b, uint32_t nq, float k, uint32_t ld_out, uint32_t *d_ids, float *d_scores,
                       uint32_t *d_counts, cudaStream_t s, const RrfRows &o = RrfRows{});

// a hybrid batch (cdb_hybrid_search_batch*): each query's kind names two of the sources dense (0), sparse (1) and TF-IDF
// (2), first list first; a source's batch holds the queries whose kind names it, in request order.  A two-source call is
// a batch of one kind.
constexpr int HYB_KIND_SRC[3][2] = {{0, 1}, {0, 2}, {1, 2}};
// "exactly two sources", then the kinds of a two-source call: nq copies of its pair's kind
cdb_status hybrid_pair_kinds(bool dense, bool sparse, bool tfidf, uint32_t nq, std::vector<uint8_t> *kinds);
// The refusals of a request that read no handle and no group, in this order: null sources; top_k > 341; null kinds, a
// kind above 2 or counts that disagree with the kinds; CDB_SEARCH_ALL_CANDIDATES with dense queries; a null handle (single
// index) or null queries of a source with queries; the sparse re-rank bound; malformed query CSR (host: host arrays).
cdb_status check_hybrid_request(const cdb_hybrid_mixed_sources *m, uint32_t nq, uint32_t top_k, bool host);
cdb_status check_hybrid_request(const cdb_hybrid_group_mixed_sources *h, uint32_t nq, uint32_t top_k, bool host);
// request positions [q0, q1): rows [row0[j], row0[j] + rows[j]) of source j's batch, n[c] queries of kind c, whose maps
// sit at map[c] in the map array: output rows (from q0), first-list rows, second-list rows (from each source's row0)
struct MixedChunk {
    uint32_t q0, q1, row0[3], rows[3], n[3];
    size_t map[3];
};
// Chunks of request positions (nq >= 1) whose lists, ld[j] columns for source j, fit in `budget` bytes, and their maps.
// A batch of one kind gets no maps: query q is row q of both its sources' batches, so the dense search writes its error
// bytes in place, and a position costs two lists and two counts.  Otherwise the maps take 3 * nq u32 and a position costs
// the widest kind present and the dense error byte.
void mixed_chunks(const uint8_t *kinds, uint32_t nq, const uint32_t ld[3], size_t budget, std::vector<MixedChunk> *chunks,
                  std::vector<uint32_t> *maps);
// one fusion launch per kind present in the chunk: lists[j] holds source j's rows of the chunk (rows unset), d_maps the map
// array on the device (null: no maps, rows in place), d_err_dense the dense search's error bytes of the chunk when there
// are maps; the outputs start at the chunk's q0, and d_err gets 0 at SPARSE_TFIDF queries
cdb_status mixed_fuse(const MixedChunk &c, const RrfList lists[3], const uint32_t *d_maps, const uint8_t *d_err_dense, float k,
                      uint32_t ld_out, uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s);

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
                             uint64_t *d_out_keys = nullptr,        // [nq][k] packed selection keys as well (shard merge)
                             const uint32_t *d_deleted = nullptr,   // deleted-row bitmap: such candidates are dropped
                             bool dedup = true);                    // report a repeated candidate once (<= 64 repeats)
// largest dimension rerank_f32_device accepts for any candidate count (its query and key buffer share 200 KB of smem)
uint32_t rerank_f32_max_dim();
// the same re-rank without truncation (top_k None): every one of the <= ncand candidates of a query is scored and sorted in
// one CTA, ncand <= RERANK_ALL_MAX_CAND; row b of the outputs is `width` wide, the first d_out_counts[b] entries best first.
// Query and keys share 200 KB of smem: dim <= (200 KB - 8 * next_pow2(ncand)) / 4, i.e. 43008 at 4096 slots.
constexpr uint32_t RERANK_ALL_MAX_CAND = 4096;
// whether rerank_all_f32_device takes this dimension and candidate count (checked before a top_k None search is enqueued)
bool rerank_all_fits(uint32_t dim, uint32_t ncand);
cdb_status rerank_all_f32_device(const float *d_raw, uint32_t pitch_elems, const float *d_raw_mags, uint64_t n_rows, uint32_t dim,
                                 const float *d_q, uint32_t q_pitch_elems, const float *d_qmags, uint32_t nq, const uint32_t *d_cand,
                                 const uint32_t *d_cand_counts, uint32_t ncand, uint32_t width, uint32_t id_base, uint32_t *d_out_ids,
                                 float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s, const uint32_t *d_labels = nullptr,
                                 uint64_t *d_out_keys = nullptr);

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
    const uint32_t *deleted;   // deleted-row bitmap (bit r = row r) or null: such rows are neither offered nor flag errors
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
};
// remove_duplicates_and_filter: ids of the entries d_ids (replica ids) or, with d_ids == null, their rows; entries with
// id == drop_id (the root) or row == CDB_INVALID_ID (pseudo nodes) are dropped; d_labels (may be null) receives the kept ids
cdb_status hnsw_dedup_device(const uint32_t *d_ids, const uint32_t *d_rows, const float *d_scores, const uint32_t *d_n, uint32_t in_cap,
                             int metric, uint32_t drop_id, uint32_t id_base, uint32_t k5, uint32_t nq, uint32_t *d_cand,
                             uint32_t *d_labels, uint32_t *d_cand_cnt, cudaStream_t s);

// ---- hnsw_warp.cu: HNSW search, one warp per query
// CDB_INVALID_PARAMS when ef_search is outside 1..4096 or the warp's shared memory (hw_carve: rows of row_pitch bytes; md: the
// metadata form with M dims) exceeds 200 KB.  Host only, so a search can refuse before it touches the device.
cdb_status hnsw_search_check(uint32_t row_pitch, uint32_t ef, bool md, uint32_t M);
cdb_status hnsw_search_warp_device(const HnswArgs &a, cudaStream_t s);
// metadata-filtered search on graphs with replica nodes
struct HnswMdArgs {
    HnswArgs a;                       // out_rows = vector row of each result (CDB_INVALID_ID for pseudo nodes)
    const uint32_t *const *node_id;   // device table [num_levels+1] of device arrays
    const uint32_t *const *node_md;
    const int32_t *md_bits;           // [n_md][M]
    const float *md_mags;
    uint32_t M;
    uint32_t pseudo_entry;
    const uint32_t *filter_offsets;   // [nq+1] rows of filter_dims per query
    const int8_t *filter_dims;        // [n_filter_rows][M]
    uint32_t n_filter_rows;
    const uint8_t *has_filter;        // [nq] (nullptr = no query has a filter)
    uint32_t *out_ids;                // [nq][out_cap] replica ids
};
// CDB_INVALID_PARAMS as hnsw_search_check
cdb_status hnsw_search_md_device(const HnswMdArgs &a, cudaStream_t s);

// ---- hnsw_build.cu
struct HnScoreCtx;
// the index's graph as the builder sees it: the search layout, the allocations that own every level array (per-level
// arrays are replaced when a level grows) and host copies of the per-level device pointers
struct GraphHost {
    GraphDev *dev;
    std::vector<void *> *allocs;
    std::vector<uint32_t> *cnt;
    std::vector<const uint32_t *> *nr, *ad, *ch;
    // graphs with replica nodes (null otherwise): host copies and device tables of the per-level node_id / node_md arrays
    std::vector<const uint32_t *> *id = nullptr, *md = nullptr;
    const uint32_t *const *id_tbl = nullptr, *const *md_tbl = nullptr;
};
// the builder's per-slot state (similarity keys, stale lowest_index, node locks), kept next to the graph it belongs to
struct HnswBuildState;
void hnsw_state_free(HnswBuildState *st);
// frees the state and the arrays that only it uses (slot keys, lowest_index, locks, list positions, and on replica graphs the
// node_id / node_md arrays and the Metadata table it grew) when `allocs` owns them; the graph's node_row / adj / child stay
void hnsw_state_release(HnswBuildState *st, std::vector<void *> *allocs);
// cdb_index_build_graph: root row n on every level, then rows [0, n) inserted
cdb_status hnsw_build_device(const HnScoreCtx &sc, uint32_t n, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0,
                             uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t seed, const GraphHost &gh,
                             HnswBuildState **out_state, cudaStream_t s, const uint32_t *d_deleted = nullptr,
                             const uint32_t *h_deleted = nullptr);
// slot state of a graph that came from elsewhere (cdb_index_set_graph), under the reload semantics of
// ProbNode::new_with_neighbors_and_versions; sc.root_row = the graph's root row
cdb_status hnsw_slot_state_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState **out_state, cudaStream_t s);
// cdb_index_insert_graph: rows [cnt[0], cnt[0] + n_new) inserted into the graph; max_level = NULL draws from `seed`;
// rows_cap bounds level 0; out_failed[n_new] may be NULL.  Every allocation precedes the first change: an error with
// *changed == false left the graph as it was, with *changed == true the graph is half-inserted and must be dropped.
cdb_status hnsw_insert_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, uint32_t n_new, const uint8_t *max_level,
                              uint64_t seed, uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t rows_cap,
                              uint8_t *out_failed, bool *changed, cudaStream_t s, const uint32_t *d_deleted = nullptr,
                              const uint32_t *h_deleted = nullptr);
// deleted-row bitmaps (d_deleted device, h_deleted host, bit r = row r; null = none): build and insert skip those rows
// (no upper-level nodes, not linked, out_failed 2)
// cdb_index_delete_rows: delete_embedding for the distinct rows rows[0..n) with the deviations D1-D4 (DESIGN.md section 4);
// out_status[i] = 0, or 2 where an Err stopped relinks.  *changed as for the insert.  The rows' nodes are looked up on the
// host; the repair is the batch loop hnsw_delete_replicas_device runs too.
cdb_status hnsw_delete_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const uint32_t *rows, uint32_t n,
                              uint32_t shortlist, uint32_t max_batch, uint8_t *out_status, bool *changed, cudaStream_t s);
// similarity keys of every slot of `level` ([cnt*nb], device)
const uint32_t *hnsw_state_slot_keys(const HnswBuildState *st, uint32_t level);
constexpr uint32_t HNSW_DELETE_EF = 512;   // the ef of a delete's traversal (vector_store.rs:1247)
// CDB_INVALID_PARAMS (with a message) when the graph writers' traversal kernel cannot run at this row pitch and ef: its
// shared memory (hw_carve, all of it dynamic) exceeds the current device's opt-in limit per block.
// The build, replica build, insert and delete entry points call it before they change anything.
cdb_status hnsw_build_smem_check(uint32_t row_pitch, uint32_t ef);

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
// cdb_index_build_graph_replicas: the main root (row main_root_row) and the pseudo root on every level, then the nodes of `rh`
// inserted as hnsw_insert_replicas_device inserts them.  gh carries the node_id / node_md tables (id_tbl / md_tbl, allocated by
// the caller); the node_row / adj / child tables are allocated here.  out_failed[n_nodes] may be NULL.  On success
// *md_bits / *md_mags point at the Metadata table and out_state is the builder's state of the replica graph, which
// hnsw_insert_replicas_device continues from.
cdb_status hnsw_build_replicas_device(const HnScoreCtx &sc, const ReplicaHost &rh, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0,
                                      uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, const GraphHost &gh,
                                      uint8_t *out_failed, const int32_t **md_bits, const float **md_mags, HnswBuildState **out_state,
                                      cudaStream_t s);
// true (and the pseudo root's row, the Metadata table's row count) when `st` is the state of a replica build
bool hnsw_state_replica_info(const HnswBuildState *st, uint32_t *pseudo_root_row, uint32_t *n_md);
// cdb_index_insert_graph_replicas: the nodes of `rh` (n_nodes entries; row already mapped to the pseudo root's row where the
// caller passed CDB_INVALID_ID; md_bits / md_mags / n_md = the table rows to append) inserted into the replica graph of
// `st`, continuing its list positions.  On success *md_bits / *md_mags point at the grown Metadata table.  *changed as for
// hnsw_insert_device.
cdb_status hnsw_insert_replicas_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const ReplicaHost &rh,
                                       uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint8_t *out_failed,
                                       const int32_t **md_bits, const float **md_mags, bool *changed, cudaStream_t s);
// cdb_index_set_graph_slot_scores: the builder's state of an uploaded graph with metadata from the similarities stored with its
// slots (scores[L] / tags[L]: host, level_counts[L] x nbrs(L); tags may be NULL), as a reference restart holds it.  The graph is
// not renumbered.  pseudo_entry == the graph's entry: no pseudo root (the state's pseudo root row is CDB_INVALID_ID).  The
// Metadata table (n_md rows) becomes the builder's.  CDB_STORAGE_MISMATCH when a filled slot's tag is not the metric's,
// CDB_INVALID_PARAMS when a level lists a node id twice; on any error nothing changed.  On success the new arrays have
// joined gh.allocs.
cdb_status hnsw_attach_replica_state_device(int metric, const GraphHost &gh, const float *const *scores, const uint8_t *const *tags,
                                            uint32_t pseudo_entry, uint32_t n_md, uint32_t md_dims, const int32_t *md_bits,
                                            const float *md_mags, HnswBuildState **out_state, cudaStream_t s);
// cdb_index_delete_rows_replicas: every node of each of the distinct rows rows[0..n) (none a root row) deleted from the replica
// graph of `st` with D1-D5 (DESIGN.md section 4); out_status[i] = 0, or 2 where an Err hit one of the row's nodes.  A row
// without a node is left alone.  *changed as for hnsw_insert_device.
cdb_status hnsw_delete_replicas_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const uint32_t *rows, uint32_t n,
                                       uint32_t shortlist, uint32_t max_batch, uint8_t *out_status, bool *changed, cudaStream_t s);

// ---- tensor_scan.cu (wgmma prefilter)
constexpr uint32_t TS_MAX_ODD = 64;   // degenerate rows that are not all-zero ride on every candidate list; more -> no prefilter
constexpr uint32_t TS_DEG_WORDS = 2 + TS_MAX_ODD;
// rows [first, first + n): d_raw / d_mags / d_out point at row `first`; rows set in d_deleted (may be null) get zero rows
cdb_status normalize_f16_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t first, uint64_t n,
                                uint32_t dim, void *d_out, uint32_t out_pitch_halfs, const uint32_t *d_deleted, cudaStream_t s);
// deleted rows: fp16 shadow rows d_rows[0..n_rows) := 0; the s8 shadow tiles d_tiles[0..n_tiles) re-quantized without the rows
// set in d_deleted (d_xs8 may be null: no s8 shadow), then *d_emax refreshed
cdb_status shadow_drop_rows_device(const uint32_t *d_rows, uint32_t n_rows, const uint32_t *d_tiles, uint32_t n_tiles, void *d_xh,
                                   uint32_t xh_pitch_halfs, const float *d_raw, uint32_t pitch_elems, const float *d_mags,
                                   uint64_t row_end, uint32_t dim, void *d_xs8, uint32_t pitch8, float2 *d_tile_se, float2 *d_tile_rcp,
                                   float *d_emax, const uint32_t *d_deleted, cudaStream_t s);
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
                               uint32_t *d_progress, float2 *d_q_se, float2 *d_q_rcp, cudaStream_t s);
// s8 form of the prefilter (DESIGN.md section 5c): shadow of the tiles touching rows [first, first + n) of rows < row_end,
// then *d_emax = max E_T over all tiles below row_end; rows set in d_deleted (may be null) are treated as degenerate
cdb_status quantize_s8_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t first, uint64_t n,
                              uint64_t row_end, uint32_t dim, void *d_xs8, uint32_t pitch8, float2 *d_tile_se, float2 *d_tile_rcp,
                              float *d_emax, const uint32_t *d_deleted, cudaStream_t s);
cdb_status tensor_scan_s8_device(const void *d_xs8, const void *d_qs8, uint32_t pitch8, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, const float2 *d_tile_se, const float2 *d_tile_rcp, const float2 *d_q_se,
                                 const float2 *d_q_rcp, uint32_t id_base, int *d_ggm,
                                 uint32_t *d_cand, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_progress, bool has_deg,
                                 int sm_count, cudaStream_t s, uint32_t *d_kept_cnt, bool *refiltered);
// d_kept_cnt (may be null): after tensor_scan_s8_kernel on a shard without degenerate or deleted rows, the candidates are
// tested again against the final bound (s8_refilter_kernel): the survivors are compacted to the front of each list and
// d_kept_cnt[q] is their number (cap for an overflowed list), *refiltered = true; d_cand_cnt keeps the emitted counts.
cdb_status tensor_scan_i8_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_ggm,
                                 uint64_t *d_cand64, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32,
                                 uint32_t *d_progress /* 2048 words */, const uint32_t *d_deleted, int sm_count, cudaStream_t s);
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
                                 uint32_t *d_ids, float *d_scores, uint32_t *d_counts, const uint32_t *d_deleted, int sm_count,
                                 cudaStream_t s, uint64_t *d_out_keys = nullptr);

}  // namespace cdb

// the results of a top_k None sparse search, in host memory: query q's entries are [off[q], off[q+1])
struct cdb_sparse_results {
    std::vector<uint64_t> off{0};
    std::vector<uint32_t> ids;
    std::vector<float> scores;
};
