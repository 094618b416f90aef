// cosdata_b200.hpp -- C++17 host-side mirror of the reference's operator surface for the distance hot
// path, header-only over the C ABI (cosdata_b200.h).  The reference is Rust; where its toolchain is absent
// this is the compiled-language host side: same names, argument meaning and error behaviour as
//   enum Storage / StorageType          src/storage/mod.rs:7-25, src/quantization/mod.rs:19-25
//   Quantization::quantize              src/quantization/mod.rs:8-17, scalar.rs:10-52
//   DistanceFunction::calculate         src/distance/mod.rs:8-22, src/models/types.rs:460-496
//   IndexOps::batch_search              src/indexes/mod.rs:260-272
//   finalize_ann_results                src/vector_store.rs:404-445
// Nothing is computed here: every method is one call into libcosdata_b200.so.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "cosdata_b200.h"

namespace cosdata {

enum class StorageType : int32_t { UnsignedByte = 0, SubByte1 = 1, SubByte2 = 2, SubByte3 = 3, HalfPrecisionFP = 4, FullPrecisionFP = 5,
                                   BFloat16 = 6 /* labelled extension, no reference variant */ };
enum class DistanceMetricKind : int32_t { Cosine = 0, Euclidean = 1, Hamming = 2, DotProduct = 3 };
enum class SearchMode : int32_t { BruteRaw = 0, BruteCodes = 1, Hnsw = 2 };

// DistanceError::{StorageMismatch, CalculationError} and the library's own failures
struct Error : std::runtime_error {
    cdb_status status;
    Error(cdb_status s, const std::string &what) : std::runtime_error(what), status(s) {}
};
struct DistanceError : Error { using Error::Error; };

inline void check(cdb_status s) {
    if (s != CDB_OK) throw Error(s, cdb_last_error_string());
}

// enum Storage: one quantized vector
struct Storage {
    StorageType storage_type;
    float mag;
    uint32_t dim;
    std::vector<uint8_t> code;  // tight layout of include/cosdata_b200.h (planes [r][ceil(D/8)] for SubByte)
};

// impl Quantization for ScalarQuantization
struct ScalarQuantization {
    int device = 0;
    Storage quantize(const std::vector<float> &v, StorageType st, std::pair<float, float> range = {-1.f, 1.f}) const {
        Storage s{st, 0.f, (uint32_t)v.size(), std::vector<uint8_t>(cdb_code_bytes((int32_t)st, (uint32_t)v.size()))};
        check(cdb_quantize_batch(device, (int32_t)st, range.first, range.second, v.data(), 1, s.dim, s.code.data(), &s.mag));
        return s;
    }
    void train(const std::vector<std::vector<float>> &) const {}  // scalar.rs:54-57
};

// HNSWIndex::sample_embedding + finalize_sampling (hnsw/mod.rs:202-351): values_range for `quantization: auto`
struct SamplingData {
    uint64_t counts[CDB_SAMPLE_COUNTERS] = {};   // above_0025 .. above_05, below_0025 .. below_05
    uint64_t values = 0;
    // sample one batch of embeddings (row-major n x dim); returns the range the reference would finalize right now
    std::pair<float, float> sample(const float *vecs, uint64_t n, uint32_t dim, float clamp_margin_percent = 1.0f, int device = 0) {
        float range[2];
        uint64_t next[CDB_SAMPLE_COUNTERS];
        check(cdb_sample_values_range(device, vecs, n, dim, clamp_margin_percent, counts, values, next, range));
        for (int i = 0; i < CDB_SAMPLE_COUNTERS; ++i) counts[i] = next[i];
        values += n * dim;
        return {range[0], range[1]};
    }
};

// prop.data: the Storage payloads of an index directory (file_persist.rs:58-108), row = record number
struct PropFile {
    uint64_t records = 0, code_bytes = 0;
    StorageType storage_type = StorageType::UnsignedByte;
    uint32_t elems = 0;
    std::vector<uint32_t> ids;
    std::vector<uint8_t> codes;
    std::vector<float> mags;
    std::vector<uint64_t> offsets;   // == ProbNode prop_value.location.0
    std::vector<uint32_t> lengths;
    explicit PropFile(const std::string &path) {
        int32_t st = -1;
        check(cdb_prop_file_scan(path.c_str(), &records, &st, &elems, &code_bytes));
        if (!records) return;
        storage_type = (StorageType)st;
        ids.resize(records); codes.resize(records * code_bytes); mags.resize(records); offsets.resize(records); lengths.resize(records);
        uint64_t got = 0;
        check(cdb_prop_file_load(path.c_str(), 0, records, ids.data(), codes.data(), mags.data(), offsets.data(), lengths.data(), &got));
    }
};

// enum DistanceMetric + impl DistanceFunction (pairwise)
struct DistanceMetric {
    DistanceMetricKind kind;
    int device = 0;
    float calculate(const Storage &x, const Storage &y) const {
        if (x.storage_type != y.storage_type) throw DistanceError(CDB_STORAGE_MISMATCH, "storage variants differ");  // cosine.rs:214
        float out = 0.f;
        int32_t st = 0;
        check(cdb_distance_pairs(device, (int32_t)kind, (int32_t)x.storage_type, x.dim, x.code.data(), &x.mag, y.code.data(), &y.mag, 1, &out, &st));
        if (st != CDB_OK) throw DistanceError(st, st == CDB_STORAGE_MISMATCH ? "StorageMismatch" : "CalculationError");
        return out;
    }
};

struct SearchResults {
    uint32_t k = 0;
    std::vector<uint32_t> ids;     // [B][k], CDB_INVALID_ID padded
    std::vector<float> scores;     // [B][k]
    std::vector<uint32_t> counts;  // [B]
    std::vector<uint8_t> err;      // [B] CDB_ERRFLAG_* (the Err the reference would return for that query)
};

// one device-resident index shard
class DenseIndex {
  public:
    DenseIndex(uint32_t dim, StorageType st, DistanceMetricKind metric, uint64_t capacity, int device = 0,
               std::pair<float, float> range = {-1.f, 1.f}, bool keep_raw_f32 = false, uint32_t id_base = 0, bool tensor_prefilter = true) {
        cdb_index_desc d{dim, (int32_t)st, (int32_t)metric, range.first, range.second, capacity, device, keep_raw_f32 ? 1 : 0, id_base,
                         tensor_prefilter ? 1u : 0u};
        check(cdb_index_create(&d, &h_));
        dim_ = dim;
    }
    ~DenseIndex() { if (h_) cdb_index_destroy(h_); }
    DenseIndex(const DenseIndex &) = delete;
    DenseIndex &operator=(const DenseIndex &) = delete;

    uint64_t size() const { return cdb_index_size(h_); }
    void append(const float *vecs, uint64_t n) { check(cdb_index_append_f32(h_, vecs, n)); }
    void set_graph(const cdb_graph_desc &g) { check(cdb_index_set_graph(h_, &g)); }

    // IndexOps::batch_search
    // all_candidates (top_k None, HNSW): every candidate, best first; k is the row width, >= (num_levels + 1) * 100
    SearchResults batch_search(const float *queries, uint32_t b, uint32_t k, SearchMode mode = SearchMode::BruteRaw,
                               uint32_t ef_search = 256, uint32_t shortlist_size = 64, bool all_candidates = false) const {
        SearchResults r;
        r.k = k;
        r.ids.resize((size_t)b * k);
        r.scores.resize((size_t)b * k);
        r.counts.resize(b);
        r.err.resize(b);
        cdb_search_params p{k, (int32_t)mode, ef_search, shortlist_size, 0, 0, all_candidates ? CDB_SEARCH_ALL_CANDIDATES : 0u, 0};
        check(cdb_search_batch(h_, queries, b, &p, r.ids.data(), r.scores.data(), r.counts.data(), r.err.data()));
        return r;
    }
    // finalize_ann_results
    std::vector<std::pair<uint32_t, float>> rerank(const float *query, const std::vector<uint32_t> &cand, uint32_t k) const {
        std::vector<uint32_t> ids(k);
        std::vector<float> sc(k);
        uint32_t n = 0;
        check(cdb_rerank_f32(h_, query, cand.data(), (uint32_t)cand.size(), k, ids.data(), sc.data(), &n));
        std::vector<std::pair<uint32_t, float>> out;
        for (uint32_t i = 0; i < n; ++i) out.emplace_back(ids[i], sc[i]);
        return out;
    }
    // index_embeddings on the device (reference defaults: config.toml:19-25); appends the root row
    void build_graph(uint32_t num_levels = 9, uint32_t nbrs = 32, uint32_t nbrs0 = 64, uint32_t ef_construction = 128,
                     uint32_t shortlist_size = 64, uint32_t max_batch = 4096, uint64_t seed = 1) {
        cdb_build_params bp{num_levels, nbrs, nbrs0, ef_construction, shortlist_size, max_batch, seed};
        check(cdb_index_build_graph(h_, &bp));
    }
    // the same for a collection with a metadata schema: preprocess_embedding's flattened IndexableEmbeddings (one entry per
    // node to create); returns the per-entry "insert would have failed" flags
    std::vector<uint8_t> build_graph_replicas(const cdb_replica_build &rb, const cdb_build_params &bp) {
        std::vector<uint8_t> failed(rb.n_nodes ? rb.n_nodes : 1);
        check(cdb_index_build_graph_replicas(h_, &bp, &rb, failed.data()));
        failed.resize(rb.n_nodes);
        return failed;
    }
    // index_embeddings on the live graph: inserts the rows appended since it was built / uploaded; max_level = the caller's
    // get_max_insert_level draws (empty: the seeded counter RNG); returns the per-row "insert failed" flags
    std::vector<uint8_t> insert_graph(const cdb_build_params &bp, const std::vector<uint8_t> &max_level = {}) {
        std::vector<uint8_t> failed(std::max<uint64_t>(cdb_index_size(h_), 1));
        uint64_t n = 0;
        check(cdb_index_insert_graph(h_, &bp, max_level.empty() ? nullptr : max_level.data(), failed.data(), &n));
        failed.resize(n);
        return failed;
    }
    // index_embeddings on a graph that build_graph_replicas built: more flattened IndexableEmbeddings (rows already appended);
    // returns the per-entry "insert failed" flags
    std::vector<uint8_t> insert_graph_replicas(const cdb_replica_insert &ri, const cdb_build_params &bp) {
        std::vector<uint8_t> failed(ri.n_nodes ? ri.n_nodes : 1);
        uint64_t n = 0;
        check(cdb_index_insert_graph_replicas(h_, &bp, &ri, failed.data(), &n));
        failed.resize(n);
        return failed;
    }
    // delete_embedding for local rows; returns the per-row status (0 deleted, 1 already deleted, 2 an Err stopped relinks)
    std::vector<uint8_t> delete_rows(const std::vector<uint32_t> &rows, uint32_t shortlist_size = 64, uint32_t max_batch = 0) {
        std::vector<uint8_t> status(std::max<size_t>(rows.size(), 1));
        check(cdb_index_delete_rows(h_, rows.data(), rows.size(), shortlist_size, max_batch, status.data(), nullptr));
        status.resize(rows.size());
        return status;
    }
    // deleted flag of every row
    std::vector<uint8_t> deleted_rows() const {
        std::vector<uint8_t> out(std::max<uint64_t>(cdb_index_size(h_), 1));
        check(cdb_index_deleted_rows(h_, 0, cdb_index_size(h_), out.data(), nullptr));
        out.resize(cdb_index_size(h_));
        return out;
    }
    // similarity of every neighbour slot of `level` (0 for empty slots), as the reference's serializer stores it
    std::vector<float> read_graph_slot_scores(uint32_t level) {
        uint32_t info[5], counts[32];
        check(cdb_index_graph_info(h_, info, counts));
        std::vector<float> out((size_t)counts[level] * (level == 0 ? info[2] : info[1]));
        check(cdb_index_read_graph_slot_scores(h_, level, out.data()));
        return out;
    }
    // delete_embedding on a graph with metadata: every node of each row (its base and Metadata replicas); per-row status
    std::vector<uint8_t> delete_rows_replicas(const std::vector<uint32_t> &rows, uint32_t shortlist_size = 64, uint32_t max_batch = 0) {
        std::vector<uint8_t> status(std::max<size_t>(rows.size(), 1));
        check(cdb_index_delete_rows_replicas(h_, rows.data(), rows.size(), shortlist_size, max_batch, status.data(), nullptr));
        status.resize(rows.size());
        return status;
    }
    // slot similarities of `level` of a graph that build_graph_replicas built
    std::vector<float> read_replica_slot_scores(uint32_t level) {
        uint32_t info[5], counts[32];
        check(cdb_index_graph_info(h_, info, counts));
        std::vector<float> out((size_t)counts[level] * (level == 0 ? info[2] : info[1]));
        check(cdb_index_read_replica_slot_scores(h_, level, out.data()));
        return out;
    }
    // raw f32 rows for rows appended as codes (cold start of a quantized index)
    void set_raw(uint64_t first_row, const float *vecs, uint64_t n) { check(cdb_index_set_raw_f32(h_, first_row, vecs, n)); }
    uint64_t raw_missing() const { return cdb_index_raw_missing(h_); }
    cdb_index *handle() const { return h_; }

  private:
    cdb_index *h_ = nullptr;
    uint32_t dim_ = 0;
};

// row-sharded search over the GPUs of one box: the library owns the NCCL communicator (SURVEY 8e)
class ShardGroup {
  public:
    // one process drives every device (a device listed twice selects the copy-based loopback gather)
    explicit ShardGroup(const std::vector<int32_t> &devices) { check(cdb_shard_group_create(devices.data(), (uint32_t)devices.size(), &g_)); }
    // one process per GPU: every rank passes the id rank 0 made with unique_id()
    ShardGroup(const std::vector<uint8_t> &id128, uint32_t world, uint32_t rank, int32_t device) {
        check(cdb_shard_group_create_rank(id128.data(), world, rank, device, &g_));
    }
    ~ShardGroup() { if (g_) cdb_shard_group_destroy(g_); }
    ShardGroup(const ShardGroup &) = delete;
    ShardGroup &operator=(const ShardGroup &) = delete;
    static std::vector<uint8_t> unique_id() {
        std::vector<uint8_t> id(CDB_NCCL_UNIQUE_ID_BYTES);
        check(cdb_nccl_unique_id(id.data()));
        return id;
    }
    void attach(uint32_t local_slot, DenseIndex &shard) { check(cdb_shard_group_attach(g_, local_slot, shard.handle())); }
    uint32_t world() const { return cdb_shard_group_world(g_); }
    // IndexOps::batch_search over all shards: one all-gather of packed keys, merged with "better score, then smaller id".
    // all_candidates (top_k None, HNSW): k is the row width, world * w with w >= every shard's (num_levels + 1) * 100
    SearchResults batch_search(const float *queries, uint32_t b, uint32_t k, SearchMode mode = SearchMode::BruteRaw,
                               uint32_t ef_search = 256, uint32_t shortlist_size = 64, bool all_candidates = false) const {
        SearchResults r;
        r.k = k;
        r.ids.resize((size_t)b * k);
        r.scores.resize((size_t)b * k);
        r.counts.resize(b);
        r.err.resize(b);
        cdb_search_params p{k, (int32_t)mode, ef_search, shortlist_size, 0, 0, all_candidates ? CDB_SEARCH_ALL_CANDIDATES : 0u, 0};
        check(cdb_search_batch_sharded(g_, queries, b, &p, r.ids.data(), r.scores.data(), r.counts.data(), r.err.data()));
        return r;
    }
    // the same with metadata filters (every shard a graph with metadata of one md_dims): filter_offsets [b + 1] index the
    // md_dims-wide i8 rows of filter_dims, has_filter[q] != 0 marks a filtered query (NULL: none); ids are replica ids
    SearchResults batch_search_filtered(const float *queries, uint32_t b, uint32_t k, const uint32_t *filter_offsets,
                                        const int8_t *filter_dims, const uint8_t *has_filter, uint32_t ef_search = 256,
                                        uint32_t shortlist_size = 64, bool all_candidates = false) const {
        SearchResults r;
        r.k = k;
        r.ids.resize((size_t)b * k);
        r.scores.resize((size_t)b * k);
        r.counts.resize(b);
        r.err.resize(b);
        cdb_search_params p{k, (int32_t)SearchMode::Hnsw, ef_search, shortlist_size, 0, 0, all_candidates ? CDB_SEARCH_ALL_CANDIDATES : 0u, 0};
        check(cdb_search_batch_filtered_sharded(g_, queries, b, &p, filter_offsets, filter_dims, has_filter, r.ids.data(), r.scores.data(),
                                                r.counts.data(), r.err.data()));
        return r;
    }
    // batch_hybrid_search over two kinds of the group's shards (host arrays in `sources`, exactly two use_* set): rows of
    // 6 * top_k columns holding the whole fused union, err = the dense search's flags (zeros without a dense source)
    SearchResults hybrid_search(const cdb_hybrid_group_sources &sources, uint32_t b, uint32_t top_k = 10,
                                float fusion_constant_k = 60.0f) const {
        SearchResults r;
        r.k = 6 * top_k;
        r.ids.resize((size_t)b * r.k);
        r.scores.resize((size_t)b * r.k);
        r.counts.resize(b);
        r.err.resize(b);
        check(cdb_hybrid_search_batch_sharded(g_, &sources, b, top_k, fusion_constant_k, r.ids.data(), r.scores.data(), r.counts.data(),
                                              r.err.data()));
        return r;
    }
    // batch_hybrid_search over a batch that mixes kinds (host arrays in `sources`, kinds[b] naming each query's pair): each
    // source searched once, rows as hybrid_search, err = the dense search's flags (0 for SPARSE_TFIDF queries)
    SearchResults hybrid_search_mixed(const cdb_hybrid_group_mixed_sources &sources, uint32_t b, uint32_t top_k = 10,
                                      float fusion_constant_k = 60.0f) const {
        SearchResults r;
        r.k = 6 * top_k;
        r.ids.resize((size_t)b * r.k);
        r.scores.resize((size_t)b * r.k);
        r.counts.resize(b);
        r.err.resize(b);
        check(cdb_hybrid_search_batch_mixed_sharded(g_, &sources, b, top_k, fusion_constant_k, r.ids.data(), r.scores.data(),
                                                    r.counts.data(), r.err.data()));
        return r;
    }

  private:
    cdb_shard_group *g_ = nullptr;
};

}  // namespace cosdata
