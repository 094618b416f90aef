/*
 * cosdata_b200.h -- C ABI of libcosdata_b200.so, the H100 (sm_90a) replacement
 * for cosdata's ANN-search distance hot path.
 *
 * The reference (cosdata/cosdata, Rust) has no FFI layer; its operator surface
 * for this path is three traits/enums.  Each entry point below names the
 * reference interface it replaces (file:line relative to the reference root)
 * and INTEGRATION.md shows the Rust `extern "C"` block + shim that binds it:
 *
 *   Quantization::quantize          src/quantization/mod.rs:8-17, scalar.rs:10-52
 *   DistanceFunction::calculate     src/distance/mod.rs:8-16, models/types.rs:469-495
 *   IndexOps::batch_search (S1)     src/indexes/mod.rs:260-272 -> hnsw/mod.rs:390-440
 *   neighbour expansion (S2)        src/vector_store.rs:1161-1191
 *   finalize_ann_results (S3)       src/vector_store.rs:404-445
 *
 * Conventions
 *   - plain C, no CUDA/torch types.  `stream` arguments are a cudaStream_t
 *     passed as void* (NULL = the handle's own stream).
 *   - every function returns cdb_status; cdb_last_error_string() describes the
 *     last failure on the calling thread.
 *   - caller owns every host buffer; the library owns device memory behind the
 *     handle.  No callbacks, no exceptions cross the ABI.
 *   - there is NO CPU fallback: without a CUDA device every compute entry
 *     point returns CDB_CUDA_ERROR.
 *   - results are defined by the reference arithmetic: integer scores and
 *     top-k ids bit-exact, f32 scores bit-identical to the reference's AVX2
 *     reduction order (DESIGN.md section 4).  Ties are broken by smaller id.
 */
#ifndef COSDATA_B200_H
#define COSDATA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CDB_ABI_VERSION 1

typedef int32_t cdb_status;
enum {
    CDB_OK = 0,
    CDB_STORAGE_MISMATCH = 1,  /* DistanceError::StorageMismatch  (src/distance/mod.rs:19) */
    CDB_CALCULATION_ERROR = 2, /* DistanceError::CalculationError (src/distance/mod.rs:20) */
    CDB_INVALID_PARAMS = 3,
    CDB_CUDA_ERROR = 4,
    CDB_NCCL_ERROR = 5,
    CDB_UNSUPPORTED = 6,       /* reference hits unimplemented!() */
    CDB_UNREACHABLE_ARM = 7    /* replica-kind pair the reference marks unreachable!() (cosine.rs:56-58, 68-70, 91-98): it would panic */
};

/* StorageType (src/quantization/mod.rs:19-25); SubByte(r) is CDB_ST_SUB1..3. */
enum {
    CDB_ST_U8 = 0,
    CDB_ST_SUB1 = 1,
    CDB_ST_SUB2 = 2,
    CDB_ST_SUB3 = 3,
    CDB_ST_F16 = 4,
    CDB_ST_F32 = 5,
    /* LABELLED EXTENSION, not a reference storage type: bfloat16 codes.  BASELINE.json configs[2] says "bf16" while the
     * reference only has IEEE f16 (StorageType::HalfPrecisionFP); this arm is what that variant would compute with
     * half::bf16 in place of half::f16 -- bf16::from_f32 rounding (nearest even, NaN keeps sign and is quieted), the same
     * sequential f32 dot product (products of two bf16 are exact in f32), the same metric arms as f16.  Parity for it is
     * defined against the oracle's restatement only. */
    CDB_ST_BF16 = 6
};
#define CDB_ST_LAST CDB_ST_BF16

/* DistanceMetric (src/models/types.rs:460-467). */
enum {
    CDB_METRIC_COSINE = 0,
    CDB_METRIC_EUCLIDEAN = 1,
    CDB_METRIC_HAMMING = 2,
    CDB_METRIC_DOT_PRODUCT = 3
};

/* search modes of cdb_search_batch */
enum {
    CDB_MODE_BRUTE_RAW = 0,   /* finalize_ann_results formula (vector_store.rs:414-439)
                                 applied to every raw f32 row: cos = dp/(|q|*|v|), no zero check */
    CDB_MODE_BRUTE_CODES = 1, /* DistanceMetric::calculate of the quantized query against every
                                 quantized row (cosine.rs:104-235 etc.); zero denominator sets
                                 err_flags[q] and skips the row */
    CDB_MODE_HNSW = 2         /* ann_search + finalize_ann_results on the uploaded graph */
};

/* per-query error flag bits (u8 err_flags[B]) */
enum {
    CDB_ERRFLAG_CALCULATION = 1, /* some scored pair had a zero denominator (cosine.rs:230-231);
                                    the reference `?`-propagates this and fails the query */
    CDB_ERRFLAG_OTHER = 2,       /* another Err of DistanceFunction::calculate */
    CDB_ERRFLAG_UNREACHABLE = 4  /* a replica-kind pair the reference marks unreachable!() was scored (the reference panics) */
};

#define CDB_INVALID_ID 0xFFFFFFFFu

typedef struct cdb_index cdb_index; /* opaque */

typedef struct {
    uint32_t dim;
    int32_t storage_type;   /* CDB_ST_* : HNSWIndex.storage_type */
    int32_t metric;         /* CDB_METRIC_* : HNSWIndex.distance_metric */
    float range_lo;         /* HNSWIndex.values_range */
    float range_hi;
    uint64_t capacity;      /* max rows resident on this device */
    int32_t device;         /* CUDA ordinal */
    int32_t keep_raw_f32;   /* keep raw f32 rows for the exact re-rank
                               (Collection.internal_to_external_map, collection.rs:110) */
    uint32_t id_base;       /* global id of local row 0 (corpus shard offset) */
    uint32_t tensor_prefilter; /* 1: also keep an fp16 copy of the L2-normalised raw rows so that large
                                  batches use the wgmma prefilter + exact re-rank (results identical) */
} cdb_index_desc;

typedef struct {
    uint32_t k;              /* top_k */
    int32_t mode;            /* CDB_MODE_* */
    uint32_t ef_search;      /* hnsw_params.ef_search   (config.toml:23) */
    uint32_t shortlist_size; /* config.search.shortlist_size (config.toml:32) */
    int32_t exact_only;      /* 1: never take a tensor-core path (pure SIMT scan); results are identical either way */
    uint32_t prefilter_k;    /* candidate slots per query of the tensor-core paths (0 = default); a query whose list
                                overflows is re-done by the exact scan on the device (alone if <= 64 queries overflow) */
    uint32_t reserved0;
    uint32_t reserved1;
} cdb_search_params;

/* ---------------------------------------------------------------- misc */
int32_t cdb_abi_version(void);
const char *cdb_last_error_string(void);
cdb_status cdb_device_count(int32_t *out);

/* Synthetic data (bench / tests): element idx of stream `seed` is
 *   z = seed + idx*0x9E3779B97F4A7C15; z = (z^(z>>30))*0xBF58476D1CE4E5B9;
 *   z = (z^(z>>27))*0x94D049BB133111EB; z ^= z>>31;
 *   value = ((int)(z>>40) - 2^23) / 2^23            (uniform on [-1,1), exact f32)
 * Row r of a dim-D matrix uses idx = r*D + c. */
cdb_status cdb_synth_fill_host(uint64_t seed, uint64_t first_idx, uint64_t n, float *out);

/* ------------------------------------------------- Quantization::quantize
 * bytes per code: u8 D | sub r*ceil(D/8) (planes [r][ceil(D/8)], plane 0 first) | f16 2D | f32 4D | bf16 2D */
size_t cdb_code_bytes(int32_t storage_type, uint32_t dim);
cdb_status cdb_quantize_batch(int32_t device, int32_t storage_type, float range_lo, float range_hi,
                              const float *vecs, uint64_t n, uint32_t dim,
                              void *out_codes, float *out_mags);

/* ---------------------- HNSWIndex::sample_embedding + finalize_sampling
 * (src/indexes/hnsw/mod.rs:202-351; `quantization: auto`, src/api/vectordb/indexes/repo.rs:41-47): count, over the
 * n*dim values of the sampled embeddings, how many exceed each threshold, then choose values_range.
 *   out_counts[0..7)  = #values >  {0.025, 0.05, 0.1, 0.2, 0.3, 0.4, 0.5}
 *   out_counts[7..14) = #values < -{0.025, 0.05, 0.1, 0.2, 0.3, 0.4, 0.5}
 *   out_range = (range_start, range_end): tightest threshold whose share (count as f32 / (n*dim) as f32 * 100) is
 *   <= clamp_margin_percent (config.toml:36, default 1.0), else -1.0 / 1.0.  NaN values count nowhere.
 * `prior_counts` (may be NULL) are added before the decision so a caller can sample in several calls like the
 * reference's per-batch sample_embedding; prior_values is the number of values they cover. */
#define CDB_SAMPLE_COUNTERS 14
cdb_status cdb_sample_values_range(int32_t device, const float *vecs, uint64_t n, uint32_t dim, float clamp_margin_percent,
                                   const uint64_t *prior_counts, uint64_t prior_values,
                                   uint64_t *out_counts, float *out_range);
/* same, d_vecs is DEVICE memory on `device`; runs on `stream` and synchronizes it before returning */
cdb_status cdb_sample_values_range_device(int32_t device, const float *d_vecs, uint64_t n, uint32_t dim, float clamp_margin_percent,
                                          const uint64_t *prior_counts, uint64_t prior_values,
                                          uint64_t *out_counts, float *out_range, void *stream);

/* ---------------------------------------------- DistanceFunction::calculate
 * (Base,Base) arm, batched over independent pairs.  out_status[i] is the
 * Result of pair i (CDB_OK / CDB_STORAGE_MISMATCH / CDB_CALCULATION_ERROR /
 * CDB_UNSUPPORTED); out[i] is defined only when it is CDB_OK. */
cdb_status cdb_distance_pairs(int32_t device, int32_t metric, int32_t storage_type, uint32_t dim,
                              const void *x_codes, const float *x_mags,
                              const void *y_codes, const float *y_mags,
                              uint64_t n_pairs, float *out, int32_t *out_status);

/* ------------------------------------------------------------ index handle */
cdb_status cdb_index_create(const cdb_index_desc *desc, cdb_index **out);
cdb_status cdb_index_destroy(cdb_index *index);
uint64_t cdb_index_size(const cdb_index *index);
cdb_status cdb_index_describe(const cdb_index *index, cdb_index_desc *out);   /* the descriptor it was created with */
/* preprocess_embedding (vector_store.rs:629-712): quantize with the index's
 * StorageType/range and append; raw rows kept when keep_raw_f32. */
cdb_status cdb_index_append_f32(cdb_index *index, const float *vecs, uint64_t n);
/* same, rows already in DEVICE memory on the index's device (n x dim f32, dense) */
cdb_status cdb_index_append_f32_device(cdb_index *index, const float *d_vecs, uint64_t n);
/* append already-quantized rows (prop.data payloads) */
cdb_status cdb_index_append_codes(cdb_index *index, const void *codes, const float *mags, uint64_t n);
/* ---- prop.data: the reference's node property file (src/models/file_persist.rs:58-108), a concatenation of serde_cbor
 * records { id: InternalId, value: Storage }; ProbNode stores each record's (FileOffset, BytesToRead)
 * (src/models/serializer/hnsw/node.rs:51-54).  Host-side readers, no GPU work:
 *   scan  -> number of records, their StorageType, elements per vector (bytes per plane for SubByte) and bytes per code in
 *            the tight layout of cdb_code_bytes(); CDB_STORAGE_MISMATCH if records differ in variant or length.
 *   load  -> records [first_record, first_record+max_records): ids, codes (tight layout), mags, and each record's byte
 *            offset/length in the file (= the node's prop_value.location).  Any out pointer may be NULL.
 *   cdb_index_append_prop_file -> append every record to the index in file order (row = record number); records must match
 *            the index's StorageType and dim (else CDB_STORAGE_MISMATCH, like the reference's calculate()). */
cdb_status cdb_prop_file_scan(const char *path, uint64_t *out_records, int32_t *out_storage_type, uint32_t *out_elems,
                              uint64_t *out_code_bytes);
cdb_status cdb_prop_file_load(const char *path, uint64_t first_record, uint64_t max_records, uint32_t *out_ids, void *out_codes,
                              float *out_mags, uint64_t *out_offsets, uint32_t *out_lengths, uint64_t *out_read);
cdb_status cdb_index_append_prop_file(cdb_index *index, const char *path, uint32_t *out_ids, uint64_t max_ids, uint64_t *out_appended);
/* Collections with a metadata schema interleave replica Metadata records { replica_id, vec: { mag, mbits } }
 * (write_prop_metadata_to_file, file_persist.rs:110-139) with the Storage records in the same file; the three functions above
 * skip them (rows = Storage records only).  These two read them: count + dimension, then ids, mags, mbits [n x md_dims] and
 * each record's byte offset / length (= NodePropMetadata.location, what a ProbNode stores). */
cdb_status cdb_prop_file_scan_metadata(const char *path, uint64_t *out_records, uint32_t *out_md_dims);
cdb_status cdb_prop_file_load_metadata(const char *path, uint64_t max_records, uint32_t md_dims, uint32_t *out_replica_ids,
                                       float *out_mags, int32_t *out_mbits, uint64_t *out_offsets, uint32_t *out_lengths,
                                       uint64_t *out_read);
/* ---- itoe.dim + itoe.<version>.data: the reference's raw-embedding store, TreeMap<InternalId, RawVectorEmbedding>
 * (src/models/collection.rs:110, 149-164; formats in src/models/serializer/tree_map/ and raw_vector_embedding.rs),
 * which finalize_ann_results reads for the exact re-rank (collection.rs:368-384).  Host-side readers, no GPU work.  Only the
 * newest state of every key counts (tree_map.rs:262-268); deleted keys and embeddings without dense values are skipped.
 *   scan -> number of live dense embeddings, their dimension, the largest internal id
 *   load -> entries [first_entry, ..) in ascending internal-id order: ids and row-major f32 vectors
 *   get  -> TreeMap::get_latest for one internal id (*out_len = 0 when absent/deleted)
 *   cdb_index_append_itoe -> cdb_index_append_f32 of every live embedding in ascending internal-id order */
cdb_status cdb_itoe_scan(const char *collection_dir, uint64_t *out_entries, uint32_t *out_dim, uint64_t *out_max_internal_id);
cdb_status cdb_itoe_load(const char *collection_dir, uint64_t first_entry, uint64_t max_entries, uint32_t *out_internal_ids,
                         float *out_vectors, uint64_t *out_read);
cdb_status cdb_itoe_get(const char *collection_dir, uint32_t internal_id, float *out_vector, uint32_t capacity, uint32_t *out_len);
cdb_status cdb_index_append_itoe(cdb_index *index, const char *collection_dir, uint32_t *out_internal_ids, uint64_t max_ids,
                                 uint64_t *out_appended);
/* Raw f32 rows for rows that were appended as codes (cdb_index_append_codes / cdb_index_append_prop_file) into a keep_raw_f32
 * index: such rows are searchable by BRUTE_CODES at once, but HNSW / BRUTE_RAW / re-rank are refused (CDB_INVALID_PARAMS)
 * until every row has its raw embedding -- what the reference reads from internal_to_external_map (collection.rs:368-384).
 *   cdb_index_set_raw_f32        rows [first_row, first_row+n) <- vecs (n x dim f32); also builds the fp16 shadow rows
 *   cdb_index_raw_missing        rows still lacking a raw embedding
 *   cdb_index_fill_raw_from_itoe row r <- embedding of internal id row_ids[r] from the itoe store (CDB_INVALID_ID = the row
 *                                has none by design, e.g. the root vector).  Cold start of a quantized on-disk index:
 *                                append_prop_file -> fill_raw_from_itoe(ids it returned) -> set_graph_from_files. */
cdb_status cdb_index_set_raw_f32(cdb_index *index, uint64_t first_row, const float *vecs, uint64_t n);
uint64_t cdb_index_raw_missing(const cdb_index *index);
cdb_status cdb_index_fill_raw_from_itoe(cdb_index *index, const char *collection_dir, const uint32_t *row_ids, uint64_t n_rows,
                                        uint64_t *out_filled, uint64_t *out_missing);
/* generate rows [first_row, first_row+n) of synthetic stream `seed` ON DEVICE and append
 * them (exactly what cdb_index_append_f32 would store for the same values) */
cdb_status cdb_index_append_synthetic(cdb_index *index, uint64_t seed, uint64_t first_row, uint64_t n);
/* copy stored state back (tests): codes/mags of rows [first, first+n) */
cdb_status cdb_index_read_codes(const cdb_index *index, uint64_t first, uint64_t n, void *out_codes, float *out_mags);

/* ---- DistanceFunction::calculate with metadata: the replica-kind arms of CosineSimilarity (src/distance/cosine.rs:34-102).
 * One side of a batch of VectorData { id: Option<&InternalId>, quantized_vec, metadata: Option<&Metadata> }
 * (src/models/types.rs:203-212): ids == NULL -> id None for all, has_id (optional) marks per-element Some/None;
 * md_bits == NULL -> metadata None for all, has_md (optional) per element; md_bits is [n x md_dims] i32 (Metadata.mbits),
 * md_mags[n] = Metadata.mag.  x is the query side (fvec_data), y the node side: kinds Pseudo/Base/Metadata follow
 * VectorData::replica_node_kind (types.rs:223-243).  out_status: CDB_OK, CDB_CALCULATION_ERROR (zero metadata or vector
 * norm product), CDB_UNREACHABLE_ARM (pairs the reference marks unreachable!()), or the storage arms' errors.  Metrics
 * other than cosine ignore the metadata, as in the reference. */
typedef struct {
    const void *codes;       /* tight layout of cdb_code_bytes() */
    const float *mags;
    const uint32_t *ids;
    const uint8_t *has_id;
    const int32_t *md_bits;
    const float *md_mags;
    const uint8_t *has_md;
} cdb_vector_data_batch;
cdb_status cdb_distance_pairs_md(int32_t device, int32_t metric, int32_t storage_type, uint32_t dim, uint32_t md_dims,
                                 const cdb_vector_data_batch *x, const cdb_vector_data_batch *y, uint64_t n_pairs,
                                 float *out, int32_t *out_status);

/* ------------------------------------------------------------ HNSW graph upload
 * Flat export of the reference's ProbNode graph (src/models/prob_node.rs:99-109): the vector of node
 * i at level L is row node_row[L][i] of the index; adjacency[L][i*nbrs(L)+s] is the level-local index
 * of the neighbour in slot s (CDB_INVALID_ID = empty slot, slot order preserved: the search examines
 * the first shortlist_size slots); child[L][i] is the level-local index one level down (L >= 1).
 * Every index must be in range (checked).  Without graph metadata level 0 holds one node per row and result ids are rows;
 * with cdb_index_set_graph_metadata several nodes may share a row.  root_row is the row holding the root vector
 * (id u32::MAX in the reference, vector_store.rs:57-67); it is never returned.  Arrays are copied. */
typedef struct {
    uint32_t num_levels;              /* hnsw_params.num_layers: levels 0..=num_levels */
    uint32_t neighbors_count;         /* slots per node, levels >= 1 (<= 64) */
    uint32_t level0_neighbors_count;  /* slots per node, level 0 (<= 64) */
    uint32_t entry;                   /* root's local index at the top level */
    uint32_t root_row;
    const uint32_t *level_counts;     /* [num_levels+1] */
    const uint32_t *const *node_row;  /* [num_levels+1] host arrays */
    const uint32_t *const *adjacency;
    const uint32_t *const *child;     /* child[0] ignored */
} cdb_graph_desc;
cdb_status cdb_index_set_graph(cdb_index *index, const cdb_graph_desc *graph);

/* ---- the reference's on-disk HNSW index (prop.data + nodes.ptr + <id>.index in one index directory; formats in
 * src/models/serializer/hnsw/{node,neighbors,latest_node}.rs) flattened into the arrays above.  The two entry links
 * (root_vec_ptr_offset, pseudo_root_vec_ptr_offset; CDB_INVALID_ID when the collection has no metadata schema) are kept by the
 * reference in LMDB next to the index parameters (src/models/types.rs:899-945) and are passed in.  Host-side, no GPU work.
 *   info8 = {num_levels, neighbors_count, level0_neighbors_count, entry, pseudo_entry, root_row, md_dims, n_md}
 *   level -> node_row (ordinal of the node's Storage record in prop.data = the row cdb_index_append_prop_file gives it),
 *            node_id (ProbNode::get_id()), node_md (metadata table row or CDB_INVALID_ID), adjacency, child
 *   cdb_index_set_graph_from_files = cdb_index_set_graph + cdb_index_set_graph_metadata (node ids are always attached so that
 *            the fixed set and the reported ids are the reference's InternalIds; searches go through the metadata-aware kernel). */
typedef struct cdb_hnsw_files cdb_hnsw_files;
cdb_status cdb_hnsw_files_open(const char *index_dir, uint32_t root_link_offset, uint32_t pseudo_root_link_offset, cdb_hnsw_files **out);
/* same for indexes written with enable_context_history: the link image is split over "<region>-<version>.ptr" files
 * (src/models/cache_loader.rs:91-113); per 8192-byte region the file with the highest version <= latest_version counts
 * (FilelessBufferManager::from_versioned, src/models/buffered_io.rs:524-570).  cdb_hnsw_files_open reads nodes.ptr when it
 * exists and otherwise this layout with latest_version = u32::MAX. */
cdb_status cdb_hnsw_files_open_versioned(const char *index_dir, uint32_t root_link_offset, uint32_t pseudo_root_link_offset,
                                         uint32_t latest_version, cdb_hnsw_files **out);
cdb_status cdb_hnsw_files_close(cdb_hnsw_files *files);
cdb_status cdb_hnsw_files_info(const cdb_hnsw_files *files, uint32_t *info8, uint32_t *level_counts);
cdb_status cdb_hnsw_files_level(const cdb_hnsw_files *files, uint32_t level, uint32_t *node_row, uint32_t *node_id, uint32_t *node_md,
                                uint32_t *adjacency, uint32_t *child);
cdb_status cdb_hnsw_files_metadata(const cdb_hnsw_files *files, int32_t *md_bits, float *md_mags);

/* Replica nodes and metadata of a graph uploaded with cdb_index_set_graph (collections with a metadata schema:
 * src/vector_store.rs:57-250, 485-712).  One embedding may own several graph nodes (its base replica and one per
 * metadata dimension set, src/models/types.rs:163-176) that share the embedding's vector row; pseudo nodes share the
 * pseudo root's row.  node_id[L][i] = ProbNode::get_id() (replica id, or prop_value.id without metadata);
 * node_md[L][i] = row of the metadata table (md_bits [n_md x md_dims] = Metadata.mbits, md_mags[n_md] = Metadata.mag) or
 * CDB_INVALID_ID when the node has no metadata; pseudo_entry = top-level index of the pseudo root
 * (HNSWIndex::get_pseudo_root_vec), the entry of every query that carries a filter (src/indexes/hnsw/mod.rs:416-420).
 * With metadata attached, results carry replica ids (as the reference's InternalSearchResult does) and
 * CDB_MODE_HNSW searches must go through cdb_search_batch_filtered. */
typedef struct {
    uint32_t md_dims, n_md;
    const int32_t *md_bits;
    const float *md_mags;
    const uint32_t *const *node_id;   /* [num_levels+1][level_counts[L]] */
    const uint32_t *const *node_md;
    uint32_t pseudo_entry;
} cdb_graph_metadata;
cdb_status cdb_index_set_graph_metadata(cdb_index *index, const cdb_graph_metadata *md);
cdb_status cdb_index_set_graph_from_files(cdb_index *index, const cdb_hnsw_files *files);
/* GPU-side index build (index_embeddings, src/vector_store.rs:714-940): appends the root vector (random in
 * values_range, id u32::MAX; vector_store.rs:57-67) as the last row and builds the HNSW graph over all rows with the
 * reference's algorithm (traverse with ef_construction per level, create_node_edges / add_neighbor with
 * lowest-similarity eviction), batches of up to max_batch vectors in flight like the reference's concurrent build.
 * The index needs capacity for one more row.  The result replaces any uploaded graph and can be read back. */
typedef struct {
    uint32_t num_levels;              /* hnsw.default_num_layer = 9 (config.toml:19-25) */
    uint32_t neighbors_count;         /* 32 */
    uint32_t level0_neighbors_count;  /* 64 */
    uint32_t ef_construction;         /* 128 */
    uint32_t shortlist_size;          /* 64 */
    uint32_t max_batch;               /* vectors inserted concurrently (0 = 4096) */
    uint64_t seed;                    /* level assignment + root vector */
} cdb_build_params;
cdb_status cdb_index_build_graph(cdb_index *index, const cdb_build_params *params);
/* The same build for a collection with a metadata schema (index_embeddings over preprocess_embedding's flattened
 * IndexableEmbeddings, src/vector_store.rs:629-780): one entry per graph node to create, in insertion order.
 *   row        vector row of the embedding; CDB_INVALID_ID = the pseudo root's vector (pseudo replicas, :655-667)
 *   node_id    ProbNode::get_id(): replica id, or prop_value.id without metadata (:803-806)
 *   base_id    prop_value.id, carried by the traversal's fvec_data (:812)
 *   md_row     row of the metadata table or CDB_INVALID_ID (prop_metadata None)
 *   max_level  the caller's get_max_insert_level draw (levels_prob, pseudo_level_probs for pseudo replicas; :749-753)
 * Nodes whose metadata has mag != 0 are indexed under the pseudo root, the rest under the main root (:461-483); edges follow
 * create_node_edges including the replica rules (:1014-1040: Metadata node <-> Pseudo neighbour only on cs == 1.0,
 * Metadata <-> Metadata not on cs == -1.0).  Appends TWO rows (main root: random in values_range, id u32::MAX, metadata
 * main_root_md; pseudo root: zeros, id u32::MAX - 257, metadata pseudo_root_md).  Every level lists [0] main root,
 * [1] pseudo root, then the created nodes in list order.  out_failed[n_nodes] (optional): 1 where the reference's insert
 * would have returned Err / panicked (the node stays unlinked).  The graph and its metadata replace any uploaded ones;
 * searches then go through cdb_search_batch_filtered / CDB_MODE_HNSW as after cdb_index_set_graph_metadata. */
typedef struct {
    uint32_t n_nodes;
    const uint32_t *row, *node_id, *base_id, *md_row;
    const uint8_t *max_level;
    uint32_t md_dims, n_md;
    const int32_t *md_bits;           /* [n_md x md_dims] Metadata.mbits */
    const float *md_mags;             /* [n_md] Metadata.mag */
    uint32_t main_root_md;            /* schema.base_dimensions() with mag 0 (vector_store.rs:79-93), or CDB_INVALID_ID */
    uint32_t pseudo_root_md;          /* schema.pseudo_root_dimensions(HIGH_WEIGHT) (vector_store.rs:185-187) */
} cdb_replica_build;
cdb_status cdb_index_build_graph_replicas(cdb_index *index, const cdb_build_params *params, const cdb_replica_build *replicas,
                                          uint8_t *out_failed);
cdb_status cdb_index_read_graph_metadata_level(const cdb_index *index, uint32_t level, uint32_t *node_id, uint32_t *node_md);
/* read the current graph back: info5 = {num_levels, neighbors_count, level0_neighbors_count, entry, root_row} */
cdb_status cdb_index_graph_info(const cdb_index *index, uint32_t *info5, uint32_t *level_counts /* [num_levels+1] or NULL */);
cdb_status cdb_index_read_graph_level(const cdb_index *index, uint32_t level, uint32_t *node_row, uint32_t *adjacency, uint32_t *child);
/* cumulative {distance evaluations, pops} of CDB_MODE_HNSW searches (roofline accounting) */
cdb_status cdb_index_hnsw_counters(const cdb_index *index, uint64_t *out2);

/* --------------------------------------------------- S1 IndexOps::batch_search
 * queries: B x dim raw f32 (search_internal quantizes them with the index's
 * storage type, hnsw/mod.rs:399-403).  out_ids/out_scores: B x k, best first;
 * unused slots get CDB_INVALID_ID / 0.  out_counts[q] = valid slots.
 * err_flags may be NULL.  k <= 1024.
 * Execution paths (same results, chosen by shape): BRUTE_RAW with an fp16 shadow, >= 4 queries, >= 16384 rows and
 * k <= 64 -> wgmma fp16 prefilter + exact re-rank; BRUTE_CODES over u8 / sub-byte codes with cosine or dot product,
 * >= 16384 rows and k <= 64 -> exact wgmma u8 scoring; everything else -> exact SIMT scan. */
cdb_status cdb_search_batch(cdb_index *index, const float *queries, uint32_t n_queries,
                            const cdb_search_params *params,
                            uint32_t *out_ids, float *out_scores, uint32_t *out_counts,
                            uint8_t *err_flags);
/* search_internal with metadata filters (src/indexes/hnsw/mod.rs:390-440, ann_search filter branch src/vector_store.rs:273-313):
 * CDB_MODE_HNSW on a graph with cdb_index_set_graph_metadata.  Query q has the filter Some(filter_dims rows
 * [filter_offsets[q], filter_offsets[q+1])) when has_filter[q] != 0 -- each row is one QueryFilterDimensions (i8 values
 * -1/0/1, md_dims wide, src/metadata/query_filtering.rs:27) -- else None (search from the main root).  has_filter == NULL
 * means no query has a filter.  err_flags: CDB_ERRFLAG_CALCULATION / CDB_ERRFLAG_UNREACHABLE (the reference would panic,
 * e.g. Some(empty list) or an unfiltered query reaching a metadata node).  out_ids are replica ids. */
cdb_status cdb_search_batch_filtered(cdb_index *index, const float *queries, uint32_t n_queries, const cdb_search_params *params,
                                     const uint32_t *filter_offsets, const int8_t *filter_dims, const uint8_t *has_filter,
                                     uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags);
/* same, every pointer is DEVICE memory on the index's device; asynchronous on `stream`.  Each search leases one of the
 * handle's scratch sets (a small pool, grown on demand): searches on different streams run concurrently, a scratch set is
 * handed to its next user only behind the event that ends its previous search. */
cdb_status cdb_search_batch_device(cdb_index *index, const float *d_queries, uint32_t n_queries,
                                   const cdb_search_params *params,
                                   uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts,
                                   uint8_t *d_err_flags, void *stream);

/* ------------------------------------- S2 neighbour expansion (gather-score)
 * score one quantized query (raw f32 in, quantized like search_internal) against
 * rows ids[0..n): DistanceMetric::calculate(query, row). */
cdb_status cdb_score_ids(cdb_index *index, const float *query, const uint32_t *ids, uint32_t n,
                         float *out, int32_t *out_status);

/* ------------------------------------------- S3 finalize_ann_results re-rank
 * exact f32 cosine of `query` against raw rows cand_ids[0..n), sorted best
 * first, truncated to k.  Needs keep_raw_f32 (or F32 storage). */
cdb_status cdb_rerank_f32(cdb_index *index, const float *query, const uint32_t *cand_ids, uint32_t n,
                          uint32_t k, uint32_t *out_ids, float *out_scores, uint32_t *out_count);

/* ------------------------------------------------ multi-GPU: row-sharded search (SURVEY 8e)
 * The reference runs IndexOps::batch_search in one process (src/indexes/mod.rs:260-272).  Here the corpus is row-partitioned
 * into one cdb_index per GPU (contiguous id ranges, cdb_index_desc.id_base = first global id of the shard); every shard
 * searches the same query batch and ONE ncclAllGather of B*k packed 64-bit keys (+ B error bytes) per rank is merged with
 * the common ordering rule (better score, then smaller id).  NCCL is bound at run time (dlopen libnccl.so.2).
 *   cdb_shard_group_create       one process drives n devices (ncclCommInitAll over device_ordinals[]); a device listed
 *                                twice selects a copy-based loopback gather (single-GPU tests of the same code path)
 *   cdb_nccl_unique_id + cdb_shard_group_create_rank   one process per GPU: rank 0 creates the id, every rank passes it in
 *   cdb_shard_group_attach       local slot i <- the shard living on that slot's device
 *   cdb_search_batch_sharded     host queries in, merged host results out (every local device gets the batch); in a
 *                                per-rank group every rank must call it with the same batch and receives the same result
 *   cdb_search_batch_sharded_device   per-rank groups only: device buffers, asynchronous on `stream`
 * Results are those cdb_search_batch would return on the concatenated corpus (exact modes), resp. the merge of the
 * per-shard HNSW results (one independent graph per shard). */
#define CDB_NCCL_UNIQUE_ID_BYTES 128
typedef struct cdb_shard_group cdb_shard_group;
cdb_status cdb_nccl_unique_id(uint8_t *out_id128);
cdb_status cdb_shard_group_create(const int32_t *device_ordinals, uint32_t n_devices, cdb_shard_group **out);
cdb_status cdb_shard_group_create_rank(const uint8_t *id128, uint32_t world, uint32_t rank, int32_t device, cdb_shard_group **out);
cdb_status cdb_shard_group_destroy(cdb_shard_group *group);
cdb_status cdb_shard_group_attach(cdb_shard_group *group, uint32_t local_slot, cdb_index *shard);
uint32_t cdb_shard_group_world(const cdb_shard_group *group);
cdb_status cdb_search_batch_sharded(cdb_shard_group *group, const float *queries, uint32_t n_queries, const cdb_search_params *params,
                                    uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags);
cdb_status cdb_search_batch_sharded_device(cdb_shard_group *group, const float *d_queries, uint32_t n_queries,
                                           const cdb_search_params *params, uint32_t *d_out_ids, float *d_out_scores,
                                           uint32_t *d_out_counts, uint8_t *d_err_flags, void *stream);

/* ------------------------------------------------ multi-GPU shard merge (5e)
 * d_ids/d_scores: [n_shards][n_queries][k] gathered per-shard results (device);
 * writes the global top-k per query with the same ordering rule. */
cdb_status cdb_merge_topk_device(int32_t device, int32_t metric, const uint32_t *d_ids, const float *d_scores,
                                 uint32_t n_shards, uint32_t n_queries, uint32_t k,
                                 uint32_t *d_out_ids, float *d_out_scores, void *stream);

/* per-phase clock64 sums of the HNSW search kernel (lane 0 of every query, summed over the queries of all searches since
 * profiling was enabled): out[0..12) = {pop + adjacency loads, fixed-set walk + compaction, issue of the row copies, wait for
 * the rows, distance chains, queue merge, end-of-level result sort, whole levels, pops, score-cache look-ups + choice of
 * speculative rows, chain phases, speculative evaluations} (the last three only with CDB_HNSW_F_SPEC); the remaining slots are 0.
 * enable != 0 zeroes the sums and switches the instrumented kernel variant on; 0 switches it off.  out (may be NULL,
 * CDB_HNSW_PROF_SLOTS entries) receives the sums accumulated so far.  Synchronizes the device. */
#define CDB_HNSW_PROF_SLOTS 16
cdb_status cdb_index_hnsw_profile(cdb_index *index, int32_t enable, uint64_t *out);
/* dense wgmma issue-rate probe (csrc/tc_probe.cu): every SM issues M128 x N256 MMAs on shared-memory-resident operands,
 * no loads, no epilogue.  kind_i8 != 0: u8 x u8 -> s32, else f16 x f16 -> f32.  out_tops = 2*M*N*K*count / time in
 * TOP/s resp. TFLOP/s: the measured roofline denominator of the integer tensor path (MEASURED_PEAKS.json only has bf16).
 * iters = 0 -> default length (~10 ms). */
cdb_status cdb_debug_tensor_peak(int32_t device, int32_t kind_i8, uint32_t iters, double *out_tops, float *out_ms);
/* measurement switch: kernel variant of CDB_MODE_HNSW searches (results are identical for every value).  Bits: 1 cooperative
 * f16 conversion, 2 next-head adjacency preload, 4 fixed-set walk through atomics, 8 round-1 CTA-per-query kernel;
 * 0xFFFFFFFF restores the default.  Process-wide. */
cdb_status cdb_debug_set_hnsw_flags(uint32_t flags);

/* ----------------------------------------------------- instrumentation
 * number of kernels launched by this library since process start (bench.py
 * reports the delta over the timed region as gpu_launches) */
uint64_t cdb_kernel_launch_count(void);
/* last search's timing of the dominant kernel, measured with CUDA events on
 * the launching stream (ms); 0 if unavailable */
cdb_status cdb_index_last_kernel_ms(const cdb_index *index, float *scan_ms, float *total_ms);
/* durations (ms) of the dominant (scan) kernel of the last min(n, 64) searches, oldest
 * first, from CUDA events recorded on the launching stream around each launch */
cdb_status cdb_index_scan_ms_history(const cdb_index *index, uint32_t n, float *out, uint32_t *out_n);
/* out4 = {searches that took a tensor-core path, of those how many needed the exact scan for some query
 * (candidate overflow / degenerate query norm), degenerate rows, 1 if an fp16 shadow exists} */
cdb_status cdb_index_stats(const cdb_index *index, uint64_t *out4);
/* the first n of: {tensor-core searches, searches where some query needed the exact scan, all-zero rows, other degenerate rows
 * (norm outside [1e-15, 1e15]: they ride on every prefilter candidate list), fp16 shadow present, queries of the LAST
 * tensor-core search that were re-done by the exact scan (candidate overflow or degenerate query norm)} */
#define CDB_STATS_FIELDS 6
cdb_status cdb_index_stats_ex(const cdb_index *index, uint64_t *out, uint32_t n);
/* candidates the prefilter emitted for each of the first n queries of the last prefilter search */
cdb_status cdb_index_last_candidate_counts(const cdb_index *index, uint32_t n, uint32_t *out);

#ifdef __cplusplus
}
#endif
#endif /* COSDATA_B200_H */
