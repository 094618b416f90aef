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
    CDB_ERRFLAG_UNREACHABLE = 4, /* a replica-kind pair the reference marks unreachable!() was scored (the reference panics) */
    CDB_ERRFLAG_BAD_FILTER = 8   /* cdb_search_batch_filtered_device: the query's filter offsets are out of order, past
                                    n_filter_rows or span more than 4096 rows; the query returns no results */
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
    uint32_t id_base;       /* global id of local row 0 (corpus shard offset); id_base + capacity <= 2^32-1 */
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
    uint32_t flags;          /* CDB_SEARCH_* bits; unknown bits are ignored */
    uint32_t reserved1;
} cdb_search_params;
/* Brute-force modes may take the tensor-core paths while the shard has deleted rows; the kernels skip those rows (the
 * fp16 / s8 prefilter shadows of a deleted row are zero and its candidates are dropped by the re-rank, the u8 wgmma masks
 * its tiles' epilogue).  Results are bit-identical with and without the flag, as with exact_only, which still wins.
 * Without it a shard with deleted rows is answered by the exact scan.  HNSW mode ignores it. */
#define CDB_SEARCH_TENSOR_WITH_DELETED 1u
/* top_k None (a dense search request without top_k, finalize_ann_results at src/vector_store.rs:404-445 with k = None):
 * every deduplicated candidate of the HNSW search is re-ranked by exact f32 cosine and the whole sorted list is returned.
 * Under the flag k is only the output row width W: row q holds counts[q] results, best first, then CDB_INVALID_ID / 0.
 *   single index (cdb_search_batch[_device], cdb_search_batch_filtered[_device]): W >= (num_levels + 1) * 100, the most
 *     candidates the traversal can report (cdb_index_graph_info gives num_levels); checked once the handle's lock is held
 *   shard groups (cdb_search_batch_sharded[_device], cdb_search_batch_filtered_sharded[_device]): W is a multiple of the
 *     world size and every local shard's (num_levels + 1) * 100 <= W / world; counts[q] is the sum over the shards.  In a
 *     per-rank group every rank must pass the same W: it sets the size of the all-gather, and a rank only checks its own
 *     shard, so a rank that refuses leaves the others waiting in the collective.  Any world size.
 * The re-rank holds the query and next_pow2((num_levels + 1) * 100) keys in 200 KB of shared memory:
 * 4 * dim + 8 * next_pow2(cap) <= 200 KB (dim <= 43008 at cap 3200).
 * Refused with CDB_INVALID_PARAMS before any device work: the flag with a CDB_MODE_BRUTE_* mode, in the dense params of
 * cdb_hybrid_search_batch[_device], W below its bound, and a dimension above that one.  Without the flag k stays in
 * 1..1024. */
#define CDB_SEARCH_ALL_CANDIDATES 2u

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
/* the MetricResult stored with each neighbour slot of `level` (serializer/hnsw/neighbors.rs:52-57, types.rs:425-431), in the
 * layout of cdb_hnsw_files_level's adjacency: out_scores[level_counts[level] x neighbours] the f32 value, out_tags the tag
 * byte (0 CosineSimilarity, 2 EuclideanDistance, 3 HammingDistance, 4 DotProductDistance); an empty slot gives 0 and 0xFF.
 * Either pointer may be NULL.  The reader does not know the index's metric, so tags are returned as stored, unchecked
 * (cdb_index_set_graph_slot_scores checks them). */
cdb_status cdb_hnsw_files_slot_scores(const cdb_hnsw_files *files, uint32_t level, float *out_scores, uint8_t *out_tags);

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
/* stored similarities per slot of the current graph, [num_levels+1] arrays of level_counts[L] x nbrs(L), in the level-local
 * order the graph was uploaded with; tags (may be NULL) are MetricResult tags and must match the index's metric.
 * Makes a graph whose metadata came from cdb_index_set_graph_metadata / cdb_index_set_graph_from_files writable: afterwards
 * cdb_index_insert_graph_replicas, cdb_index_delete_rows_replicas and cdb_index_read_replica_slot_scores accept it.  The
 * builder's state is the one the reference holds after a restart (ProbNode::new_with_neighbors_and_versions,
 * prob_node.rs:145-181): every filled slot keeps its stored similarity, lowest_index is derived afresh (the first empty slot,
 * else the first slot with the strictly lowest similarity).  The graph is not renumbered: searches and
 * cdb_index_read_graph_level see the same arrays before and after.  The roots keep their indices; a loaded node's list
 * position (the order in which a deleted row's nodes repair, D5) is the level-0 index of its node in the uploaded order, and
 * nodes inserted later follow every loaded node.  The graph's Metadata table becomes the builder's (md_bits_new appends to it).
 * A graph whose pseudo_entry is its entry has no pseudo root (a collection without a metadata schema, as
 * cdb_index_set_graph_from_files uploads it): its inserts refuse pseudo replicas (row CDB_INVALID_ID) and nodes whose
 * Metadata has mag != 0, and its deletes refuse only the main root's row.
 * Refusals, nothing changed and the graph stays searchable: a filled slot whose tag is not the metric's MetricResult variant
 * (cosine 0, dot product 4, Euclidean 2, Hamming 3): CDB_STORAGE_MISMATCH; no graph, a graph without metadata (a
 * cdb_index_set_graph graph derives its state itself), a graph that already has its builder state (a replica build or an
 * earlier call), a null level array, or a level listing a node id twice: CDB_INVALID_PARAMS.  Takes the writer lock;
 * searches enqueued before the call finish first.  Every device allocation happens before anything changes. */
cdb_status cdb_index_set_graph_slot_scores(cdb_index *index, const float *const *scores, const uint8_t *const *tags);
/* GPU-side index build (index_embeddings, src/vector_store.rs:714-940): appends the root vector (random in
 * values_range, id u32::MAX; vector_store.rs:57-67) as the last row and builds the HNSW graph over all rows with the
 * reference's algorithm (traverse with ef_construction per level, create_node_edges / add_neighbor with
 * lowest-similarity eviction), batches of up to max_batch vectors in flight like the reference's concurrent build.
 * The index needs capacity for one more row.  The result replaces any uploaded graph and can be read back.
 * The traversal keeps a row and ef_construction queue entries in shared memory: a row size / ef_construction pair above the
 * device's per-block limit (on an H100, f32 rows at ef_construction 4096 fit up to about D = 10.4K) is refused with CDB_INVALID_PARAMS
 * before anything changes; the same check guards the replica build, the insert and the delete (at ef 512). */
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
 * searches then go through cdb_search_batch_filtered / CDB_MODE_HNSW as after cdb_index_set_graph_metadata.  The handle
 * keeps the builder's state, so cdb_index_insert_graph_replicas can grow the graph later. */
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
/* GPU-side index_embeddings on the current graph (src/vector_store.rs:714-940): inserts every row appended since the graph
 * was built / uploaded, i.e. rows [level_counts[0], cdb_index_size()), in ascending row order, with the same traversal and
 * create_node_edges / add_neighbor as cdb_index_build_graph (which is this insert applied to a graph holding only the root).
 * params->num_levels / neighbors_count / level0_neighbors_count must equal the graph's (else CDB_INVALID_PARAMS);
 * ef_construction, shortlist_size, max_batch as for the build, batches of max(1, min(max_batch, rows already linked / 8));
 * max_batch = 1 inserts one row at a time (deterministic).  max_level[n_new] (may be NULL): the caller's
 * get_max_insert_level draws, clamped to num_levels; NULL = the build's counter RNG on the row index with params->seed.
 * out_failed[n_new] (may be NULL): 1 where the reference's insert returns Err (the node stays unlinked).
 * Each node keeps the add_neighbor state of the reference: a similarity per slot and a lowest_index that eviction leaves
 * stale.  A graph built on this handle keeps its state in memory; a graph from cdb_index_set_graph gets it derived on the
 * first insert as the reference derives it when it loads nodes from storage (ProbNode::new_with_neighbors_and_versions,
 * prob_node.rs:145-181: every slot's similarity recomputed, lowest_index = the first empty slot, else the first slot with
 * the strictly lowest similarity).  A slot whose pair is an Err (e.g. a zero-norm row under cosine) gets MetricResult::min
 * and is the first slot replaced.  Graphs with metadata (cdb_index_set_graph_metadata, *_replicas, *_from_files):
 * CDB_UNSUPPORTED (a graph that cdb_index_build_graph_replicas built grows through cdb_index_insert_graph_replicas).  No new rows: CDB_OK, *out_inserted = 0.  The level-0 list must be rows 0..level_counts[0]-1.
 * Takes the writer lock; searches enqueued (cdb_search_batch_device) before the call see the old graph, searches after it
 * the new one; the call returns once the graph is complete.  Failure: every device allocation happens before the graph
 * changes, so an error there (e.g. CDB_CUDA_ERROR on out-of-memory) leaves the graph and its rows as they were and the call
 * can be repeated.  An error after the graph started changing (a failed kernel or copy) drops the graph: the index has none
 * until cdb_index_build_graph / cdb_index_set_graph, and cdb_last_error_string says so. */
cdb_status cdb_index_insert_graph(cdb_index *index, const cdb_build_params *params, const uint8_t *max_level, uint8_t *out_failed,
                                  uint64_t *out_inserted);
/* index_embeddings on a graph with metadata (src/vector_store.rs:714-780): creates more nodes of preprocess_embedding's
 * flattened IndexableEmbeddings (:629-712) in a graph that cdb_index_build_graph_replicas built on this handle and that
 * earlier calls of this function may have grown.  The replica build, continued:
 *   row        a row < cdb_index_size() the caller has already appended, or CDB_INVALID_ID for the pseudo root's row (pseudo
 *              replicas, :655-667); a row out of range, one of the graph's two root rows or a deleted row: CDB_INVALID_PARAMS
 *   node_id, base_id, md_row, max_level   as in cdb_replica_build; md_row is CDB_INVALID_ID or below the table's rows plus
 *              n_md_new; max_level is required when n_nodes > 0 (clamped to num_levels)
 *   md_dims    must equal the graph's
 *   n_md_new, md_bits_new, md_mags_new   rows appended to the graph's Metadata table, only when the call returns CDB_OK
 * A node whose metadata has mag != 0 descends from the pseudo root, every other node from the main root; edges follow
 * create_node_edges with the replica rules (:1014-1040), and every node keeps its add_neighbor state (slot similarities,
 * stale lowest_index) from the build and earlier inserts.  New nodes are appended to every level they reach, behind the
 * existing ones, in list order.  out_failed[n_nodes] (may be NULL): 1 where the reference's insert returns Err (the node
 * stays unlinked).  *out_inserted (may be NULL) = n_nodes.
 * params: num_levels / neighbors_count / level0_neighbors_count must equal the graph's; ef_construction, shortlist_size and
 * max_batch as for the build (batches of max(1, min(max_batch, nodes already linked / 8)); 1 inserts one node at a time,
 * deterministically); seed is unused (level draws come from the caller).
 * No graph, or a graph without metadata (those grow through cdb_index_insert_graph): CDB_INVALID_PARAMS.  A graph whose
 * metadata came from cdb_index_set_graph_metadata / cdb_index_set_graph_from_files: CDB_UNSUPPORTED (its slot similarities
 * cannot be derived) until cdb_index_set_graph_slot_scores attached the stored ones; from then on it grows like a graph
 * built here.  A graph without a pseudo root refuses pseudo replicas and nodes whose Metadata has mag != 0
 * (CDB_INVALID_PARAMS).  n_nodes == 0: CDB_OK, *out_inserted = 0, nothing changes (no table rows are appended either).
 * Locking, the order against enqueued searches and the failure contract are those of cdb_index_insert_graph: every
 * allocation comes before the graph changes, so an allocation failure leaves the graph, its metadata and its table as they
 * were; an error after the graph started changing drops the graph and its metadata, and cdb_last_error_string says so.
 * cdb_index_insert_graph, cdb_index_delete_rows and cdb_index_read_graph_slot_scores stay CDB_UNSUPPORTED on these graphs;
 * they delete through cdb_index_delete_rows_replicas and read slot scores through cdb_index_read_replica_slot_scores. */
typedef struct {
    uint32_t n_nodes;                           /* graph nodes to create, in insertion order */
    const uint32_t *row, *node_id, *base_id, *md_row;   /* as in cdb_replica_build */
    const uint8_t *max_level;                   /* the caller's get_max_insert_level draws */
    uint32_t md_dims;                           /* must equal the graph's */
    uint32_t n_md_new;                          /* rows appended to the graph's Metadata table */
    const int32_t *md_bits_new;                 /* [n_md_new x md_dims] */
    const float *md_mags_new;                   /* [n_md_new] */
} cdb_replica_insert;
cdb_status cdb_index_insert_graph_replicas(cdb_index *index, const cdb_build_params *params, const cdb_replica_insert *nodes,
                                           uint8_t *out_failed, uint64_t *out_inserted);
/* similarity stored with each neighbour slot of `level` (level_counts[level] x neighbours f32, the MetricResult value; 0 for
 * empty slots): what the reference's serializer writes next to each link (serializer/hnsw/neighbors.rs:53-57).  Derived
 * as above for an uploaded graph.  Graphs with metadata: CDB_UNSUPPORTED. */
cdb_status cdb_index_read_graph_slot_scores(cdb_index *index, uint32_t level, float *out_scores);
/* delete_embedding (src/vector_store.rs:1206-1371) for local rows rows[0..n) (row numbers as cdb_score_ids takes them: a shard
 * caller subtracts id_base).  A row out of range or the graph's root_row: CDB_INVALID_PARAMS, nothing changed.
 * out_status[n] (may be NULL): 0 deleted; 1 already deleted (by an earlier call or earlier in this list), nothing happened;
 * 2 deleted and unlinked, but a traversal or rescoring Err stopped some relinks (D3).  *out_deleted (may be NULL) = rows
 * newly deleted.  Per level, top-down: the deleted node D's stored codes traverse from the root with nothing pre-inserted
 * in the fixed set, ef = 512 (the reference's literal) and the best 100 kept; remove_neighbor_by_id(D) on each of D's
 * neighbours in slot order (lowest_index left stale); a neighbour whose list emptied is relinked: the results minus D and
 * itself, rescored against it, sorted best first (ties: smaller id), through create_node_edges / add_neighbor with its
 * stale lowest_index.  shortlist_size = config.search.shortlist_size; max_batch (0 = 4096) deletes in flight, each batch
 * traversing the graph as of its start; 1 deletes one row at a time in list order (deterministic).  Deviations:
 *   D1 D is unlinked on every level it is on, whether or not the traversal found it (a deleted row never comes back from a
 *      search); where it was not found there is nothing to take out of the results.
 *   D2 links to D from nodes outside D's list are cleared too (the reference leaves them dangling): after D's own slots,
 *      one pass clears every slot naming D, then each node it cleared a slot of is relinked, in ascending level-local
 *      index, if its list is empty at its turn.  In batched mode relink candidates exclude rows deleted in the batch.
 *   D3 an Err stops relinks, not unlinking: a failed traversal stops the relinks of that level and the levels below, a
 *      rescoring Err that one relink; D is unlinked everywhere and gets status 2.
 *   D4 D keeps its node entries with an empty adjacency on every level (an isolated node); rows are never reused.
 * Deleted rows: the exact scans never return them nor flag their errors; the tensor-core brute-force paths are bypassed
 * while any row is deleted (the exact scan answers) unless the search sets CDB_SEARCH_TENSOR_WITH_DELETED, which lets them
 * run and skip the deleted rows (same results; making that the default is a later behaviour change).  The
 * call zeroes the deleted rows' fp16 shadow rows and re-quantizes the s8 shadow tiles they are in, without them;
 * cdb_index_build_graph / cdb_index_insert_graph skip them (out_failed
 * 2, no nodes above level 0), cdb_index_build_graph_replicas refuses a list naming one, cdb_index_set_graph refuses a
 * graph linking one.  cdb_score_ids, cdb_rerank_f32 and cdb_distance_pairs take explicit ids and are unchanged.  Without
 * a graph the call only marks the rows.  Graphs with metadata: CDB_UNSUPPORTED, nothing changed.  Locking, the order
 * against enqueued searches and the failure contract are those of cdb_index_insert_graph; the marks are set only once the
 * repair has succeeded. */
cdb_status cdb_index_delete_rows(cdb_index *index, const uint32_t *rows, uint64_t n, uint32_t shortlist_size, uint32_t max_batch,
                                 uint8_t *out_status, uint64_t *out_deleted);
/* delete_embedding on a graph that cdb_index_build_graph_replicas built, or whose stored slot similarities
 * cdb_index_set_graph_slot_scores attached (and cdb_index_insert_graph_replicas may have grown).
 * The unit is a vector row (one embedding): deleting row r deletes every graph node whose node_row is r -- its base replica
 * and all of its Metadata replicas, on every level.  Arguments, out_status, *out_deleted, the marks and the deleted rows'
 * treatment elsewhere are those of cdb_index_delete_rows; a status is per row (2 if an Err hit any of its nodes).  A row
 * with no graph node (appended after the build, or never listed) is only marked; a row whose insert failed has isolated
 * nodes and is traversed and marked like any other.  D1-D4 apply to each node R of the row, with
 *   D5 replica rules.  R traverses as the graph sees it: R's vector row, R's Metadata row and Some(R's node_id) (that id only
 *      decides the Pseudo kind, which a data row's replicas never have), from the pseudo root when its metadata has
 *      mag != 0, else from the main root, nothing pre-inserted, ef 512, best 100 kept.  A base replica's traversal is the
 *      reference's own (a Base-kind query from the main root).  An emptied neighbour N is relinked from R's results minus R,
 *      N and every node of a row deleted in the batch, rescored with the replica arms (calculate(N, candidate), N's id and
 *      metadata as x), sorted best first (ties: smaller id), then create_node_edges with the replica edge rules (cosine: a
 *      Metadata N takes a Pseudo neighbour only at cs == 1.0, two Metadata nodes never link at cs == -1.0).  A rescoring Err,
 *      CDB_UNREACHABLE_ARM included (a Pseudo N rescoring a Metadata candidate), stops that relink (D3).  Order: all nodes of
 *      a batch traverse the graph as of the batch's start; per level, a row's nodes repair their own slots in list order;
 *      then the D2 sweep over all of the batch's nodes, after which each touched node is relinked from the candidates of
 *      the first deleted node (in list order) it named.  max_batch = 1 deletes one row at a time in list order
 *      (deterministic); larger batches guarantee the invariants only.
 * Refusals (nothing changes, no marks): a row out of range, the main root's or the pseudo root's row (pseudo replicas share
 * it), shortlist_size outside 1..64, no graph or a graph without metadata (cdb_index_delete_rows): CDB_INVALID_PARAMS; a
 * graph whose metadata came from cdb_index_set_graph_metadata / cdb_index_set_graph_from_files without
 * cdb_index_set_graph_slot_scores: CDB_UNSUPPORTED.  Locking, the order against enqueued searches and the failure contract are those of cdb_index_insert_graph_replicas: an error after
 * the graph started changing drops the graph and its metadata. */
cdb_status cdb_index_delete_rows_replicas(cdb_index *index, const uint32_t *rows, uint64_t n, uint32_t shortlist_size,
                                          uint32_t max_batch, uint8_t *out_status, uint64_t *out_deleted);
/* the slot similarities a replica build, insert or delete keeps for `level` (layout and values as in
 * cdb_index_read_graph_slot_scores; on a Pseudo-Metadata edge both slots hold calculate(Metadata end, Pseudo end)).  A graph
 * without metadata: CDB_INVALID_PARAMS; uploaded metadata without cdb_index_set_graph_slot_scores: CDB_UNSUPPORTED. */
cdb_status cdb_index_read_replica_slot_scores(cdb_index *index, uint32_t level, float *out_scores);
/* out[i] = 1 if row first+i is deleted (first + n <= capacity); *out_total = deleted rows of the index (either pointer may be
 * NULL when unused) */
cdb_status cdb_index_deleted_rows(const cdb_index *index, uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total);
/* cumulative {distance evaluations, pops} of CDB_MODE_HNSW searches (roofline accounting) */
cdb_status cdb_index_hnsw_counters(const cdb_index *index, uint64_t *out2);

/* --------------------------------------------------- S1 IndexOps::batch_search
 * queries: B x dim raw f32 (search_internal quantizes them with the index's
 * storage type, hnsw/mod.rs:399-403).  out_ids/out_scores: B x k, best first;
 * unused slots get CDB_INVALID_ID / 0.  out_counts[q] = valid slots.
 * err_flags may be NULL.  k <= 1024 (CDB_SEARCH_ALL_CANDIDATES: every candidate, k = the row width).
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
/* same, every pointer is DEVICE memory on the index's device; asynchronous on `stream` (NULL: the handle's own stream) and
 * re-entrant through the scratch pool like cdb_search_batch_device.  d_filter_dims holds n_filter_rows rows of md_dims i8
 * values; d_filter_offsets [n_queries + 1] index those rows.  d_out_counts and d_err_flags may be NULL.
 * Refused with CDB_INVALID_PARAMS before any device work: a null handle, params, queries or outputs (n_queries > 0), a mode
 * other than CDB_MODE_HNSW, k outside 1..1024, d_has_filter without d_filter_offsets, n_filter_rows > 0 without
 * d_filter_dims, and d_has_filter on a graph without metadata (d_has_filter == NULL there runs the plain HNSW search).
 * The host cannot read the offsets: a filtered query whose range is not off[q] <= off[q+1] <= n_filter_rows with at most
 * 4096 rows gets CDB_ERRFLAG_BAD_FILTER and count 0, and no row outside [0, n_filter_rows) is read. */
cdb_status cdb_search_batch_filtered_device(cdb_index *index, const float *d_queries, uint32_t n_queries,
                                            const cdb_search_params *params, const uint32_t *d_filter_offsets,
                                            const int8_t *d_filter_dims, uint32_t n_filter_rows, const uint8_t *d_has_filter,
                                            uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts,
                                            uint8_t *d_err_flags, void *stream);
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
 * first, truncated to k.  Needs keep_raw_f32 (or F32 storage).  A candidate listed
 * more than once is reported once per listing, as finalize_ann_results reports it.
 * An id outside [id_base, id_base + size) is refused with CDB_INVALID_PARAMS before
 * any device work. */
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
 *   cdb_shard_group_attach       local slot i <- the shard living on that slot's device.  CDB_INVALID_PARAMS, nothing
 *                                attached, unless the shard has the dimension, metric and storage type of every shard
 *                                already attached to another local slot and its [id_base, id_base + capacity) meets
 *                                none of theirs (checked whatever the attach order)
 *   cdb_search_batch_sharded     host queries in, merged host results out (every local device gets the batch); in a
 *                                per-rank group every rank must call it with the same batch and receives the same result
 *   cdb_search_batch_sharded_device   per-rank groups only: device buffers, asynchronous on `stream`
 * Both searches refuse world * k * 8 > 200 KB (the merge's shared memory) with CDB_INVALID_PARAMS before any copy or
 * search is issued.  Under CDB_SEARCH_ALL_CANDIDATES (HNSW) that bound does not apply: each rank's sorted list fills
 * k / world columns and the lists are merged without truncation, the batch in chunks that keep the gather within 256 MB.
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
/* cdb_search_batch_filtered over a shard group: every shard runs its own filtered HNSW search (from its own pseudo root for a
 * filtered query) and the results are merged like cdb_search_batch_sharded's, error bytes OR-ed over the ranks.  The filter
 * arguments are those of cdb_search_batch_filtered (host form: queries and filter CSR go to every local device) and of
 * cdb_search_batch_filtered_device (device form: per-rank groups only, like cdb_search_batch_sharded_device; every rank
 * passes the same batch and filters, and a bad filter range gives CDB_ERRFLAG_BAD_FILTER and count 0).  Every local shard
 * must have graph metadata with the same md_dims, checked at search time (metadata may be attached after
 * cdb_shard_group_attach): CDB_INVALID_PARAMS otherwise.  out_ids are replica ids. */
cdb_status cdb_search_batch_filtered_sharded(cdb_shard_group *group, const float *queries, uint32_t n_queries,
                                             const cdb_search_params *params, const uint32_t *filter_offsets, const int8_t *filter_dims,
                                             const uint8_t *has_filter, uint32_t *out_ids, float *out_scores, uint32_t *out_counts,
                                             uint8_t *err_flags);
cdb_status cdb_search_batch_filtered_sharded_device(cdb_shard_group *group, const float *d_queries, uint32_t n_queries,
                                                    const cdb_search_params *params, const uint32_t *d_filter_offsets,
                                                    const int8_t *d_filter_dims, uint32_t n_filter_rows, const uint8_t *d_has_filter,
                                                    uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts,
                                                    uint8_t *d_err_flags, void *stream);

/* ------------------------------------------------ multi-GPU shard merge (5e)
 * d_ids/d_scores: [n_shards][n_queries][k] gathered per-shard results (device);
 * writes the global top-k per query with the same ordering rule. */
cdb_status cdb_merge_topk_device(int32_t device, int32_t metric, const uint32_t *d_ids, const float *d_scores,
                                 uint32_t n_shards, uint32_t n_queries, uint32_t k,
                                 uint32_t *d_out_ids, float *d_out_scores, void *stream);

/* per-phase clock64 sums of the HNSW search kernel (lane 0 of every query, summed over the queries of all searches since
 * profiling was enabled): out[0..9) = {pop + adjacency loads, fixed-set walk + compaction, issue of the row copies, wait for
 * the rows, distance chains, candidate-pool update (append, next head, trim), end-of-level result sort, whole levels, pops},
 * then out[9] = pool trims and out[10] = trims that fell back to an exact selection (counts); the remaining slots are 0.
 * enable != 0 zeroes the sums and switches the instrumented kernel variant on; 0 switches it off.  out (may be NULL,
 * CDB_HNSW_PROF_SLOTS entries) receives the sums accumulated so far.  Synchronizes the device. */
#define CDB_HNSW_PROF_SLOTS 16
cdb_status cdb_index_hnsw_profile(cdb_index *index, int32_t enable, uint64_t *out);
/* dense wgmma issue-rate probe (csrc/tc_probe.cu): every SM issues M128 x N256 MMAs on shared-memory-resident operands,
 * no loads, no epilogue.  kind_i8 != 0: u8 x u8 -> s32, else f16 x f16 -> f32.  out_tops = 2*M*N*K*count / time in
 * TOP/s resp. TFLOP/s: the measured roofline denominator of the integer tensor path (MEASURED_PEAKS.json only has bf16).
 * iters = 0 -> default length (~10 ms). */
cdb_status cdb_debug_tensor_peak(int32_t device, int32_t kind_i8, uint32_t iters, double *out_tops, float *out_ms);
/* the BM25 idf arithmetic (csrc/bm25_idf.h) as the library runs it, so that a binding can check its bits against the
 * platform's log1pf (f32::ln_1p): bm25_log1pf(x[i]) -> out_log1p[i] for i < n, and
 * bm25_idf(n_docs[j], df[j]) -> out_idf[j] for j < n_pairs.  on_device != 0: the device copy the idf kernels inline, every
 * pointer a device pointer on the current device, enqueued on `stream` (NULL = the legacy default stream), asynchronous.
 * on_device == 0: the same source compiled for the host (no search runs it), host pointers, synchronous (stream unused). */
cdb_status cdb_debug_bm25(int32_t on_device, const float *x, uint64_t n, float *out_log1p, const uint32_t *n_docs,
                          const uint32_t *df, uint64_t n_pairs, float *out_idf, void *stream);
/* former measurement switch of CDB_MODE_HNSW kernel variants.  HNSW search now has one kernel per graph kind, so every value
 * is accepted and selects nothing; the entry point stays for callers built against it. */
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
 * tensor-core search that were re-done by the exact scan (candidate overflow or degenerate query norm), tensor-core
 * searches whose prefilter ran in the s8 form (also counted in the first field), tensor-core searches that ran while the
 * shard had deleted rows (CDB_SEARCH_TENSOR_WITH_DELETED; also counted in the first field)} */
#define CDB_STATS_FIELDS 8
cdb_status cdb_index_stats_ex(const cdb_index *index, uint64_t *out, uint32_t n);
/* candidates the prefilter emitted for each of the first n queries of the last prefilter search */
cdb_status cdb_index_last_candidate_counts(const cdb_index *index, uint32_t n, uint32_t *out);

/* ------------------------------------------------ sparse inverted index
 * InvertedIndex (src/indexes/inverted/mod.rs): SPLADE-style sparse vectors, a list of (dim u32, value f32) pairs per row.
 * Rows are CSR: row r holds pairs [row_offsets[r], row_offsets[r+1]) and has id id_base + r.  Every pair is indexed under
 * key = quantize(value) = (((value / values_upper_bound) * max).clamp(0, max) as u8).min(max), max = 2^bits - 1, zero and
 * duplicate pairs included (inverted_index.rs:168-172).  Empty rows are allowed and never candidates.
 * A search is SparseAnnQueryBasic::sequential_search (sparse_ann_query.rs:68-147): every query pair whose dim has a list
 * adds qv * key (u32, wrapping) to each live row of the visited keys (all keys when qv > low, else keys >= etv, with
 * etv = ((2^bits * thr).min(255.0)) as u8 and low = (thr * 2^bits) as u32); a row is a candidate once any visited list holds
 * it.  The best k * f candidates are kept (higher similarity, then smaller id; f = reranking_factor when rerank, else 1).
 *   rerank = 0: out_scores = similarity as f32, best first.
 *   rerank = 1: finalize_sparse_ann_results (inverted/mod.rs:331-381) -- dp = 0f32; dp += row_value * query_value over the
 *               query pairs in the caller's order (a row's last pair of a dim wins, dims the row lacks are skipped), sorted
 *               by total_cmp (NaN canonicalised to the sign-set quiet NaN), ties to the smaller id, truncated to k.
 * out_counts[q] = min(k, candidates); unused slots hold CDB_INVALID_ID / 0.  k must be 1..1024 and k * f <= 5120
 * (CDB_INVALID_PARAMS otherwise, nothing truncated); top_k None (k = 0) is cdb_sparse_search_batch_all.  Searches on one handle are re-entrant; append and delete take the
 * handle exclusively and first wait for the searches already enqueued on the device.  An append that fails changes nothing.  Deleted rows (a tombstone per row, as mark_embedding_as_deleted with the inserted pairs leaves it)
 * are never candidates; rows are not reused.  Without a CUDA device every compute entry point returns CDB_CUDA_ERROR. */
typedef struct cdb_sparse_index cdb_sparse_index; /* opaque */

typedef struct {
    int32_t device;
    uint32_t quantization_bits;   /* 4..8 (QuantizationBits, src/api/vectordb/indexes/dtos.rs:18-25; default 4) */
    float values_upper_bound;     /* InvertedIndex.values_upper_bound (1.0 before sampling) */
    uint64_t capacity_rows;       /* id_base + capacity_rows <= 2^32 - 1 */
    uint64_t capacity_pairs;      /* (dim, value) pairs over all rows */
    uint32_t id_base;
} cdb_sparse_index_desc;

typedef struct {
    uint32_t k;                        /* top_k: 1..1024 for cdb_sparse_search_batch{,_device}; 0 = None, which only
                                          cdb_sparse_search_batch_all takes (reranking_factor is then ignored) */
    float early_terminate_threshold;   /* the request's value, else config.search.early_terminate_threshold (0.0) */
    int32_t rerank;                    /* config.rerank_sparse_with_raw_values (default 0) */
    uint32_t reranking_factor;         /* config.sparse_raw_values_reranking_factor (default 5), used when rerank */
} cdb_sparse_search_params;

cdb_status cdb_sparse_index_create(const cdb_sparse_index_desc *desc, cdb_sparse_index **out);
cdb_status cdb_sparse_index_destroy(cdb_sparse_index *index);
uint64_t cdb_sparse_index_size(const cdb_sparse_index *index);
/* n rows; row_offsets[n+1] (row_offsets[0] = 0), dims / values [row_offsets[n]] */
cdb_status cdb_sparse_index_append(cdb_sparse_index *index, const uint64_t *row_offsets, const uint32_t *dims, const float *values,
                                   uint64_t n);
/* tombstones rows[0..n) (local rows < cdb_sparse_index_size; deleting a row twice is a no-op) */
cdb_status cdb_sparse_index_delete_rows(cdb_sparse_index *index, const uint32_t *rows, uint64_t n);
/* out[i] = 1 if row first+i is deleted (first + n <= capacity_rows); *out_total = deleted rows (either may be NULL) */
cdb_status cdb_sparse_index_deleted_rows(const cdb_sparse_index *index, uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total);
/* B queries as CSR (q_offsets[B+1]); out_ids / out_scores [B][k], out_counts [B] */
cdb_status cdb_sparse_search_batch(cdb_sparse_index *index, const uint64_t *q_offsets, const uint32_t *q_dims, const float *q_values,
                                   uint32_t n_queries, const cdb_sparse_search_params *params, uint32_t *out_ids, float *out_scores,
                                   uint32_t *out_counts);
/* same with every array in DEVICE memory on the index's device, asynchronous on `stream` (NULL = the legacy default stream) */
cdb_status cdb_sparse_search_batch_device(cdb_sparse_index *index, const uint64_t *d_q_offsets, const uint32_t *d_q_dims,
                                          const float *d_q_values, uint32_t n_queries, const cdb_sparse_search_params *params,
                                          uint32_t *d_ids, float *d_scores, uint32_t *d_counts, void *stream);
/* top_k None (SparseSearchRequestDto.top_k omitted): sequential_search keeps every candidate and finalize_sparse_ann_results
 * re-ranks and sorts all of them without truncating (sparse_ann_query.rs:136-145, inverted/mod.rs:331-381).  params->k must
 * be 0 (else CDB_INVALID_PARAMS); reranking_factor is ignored; the threshold and rerank keep their meaning above.
 *   candidates: exactly the rows the top-k search considers -- live rows touched by any visited list, rows reached only
 *               through zero products included, deleted and empty rows never; the similarity is the same wrapping u32.
 *   rerank = 0: every candidate with score = similarity as f32, ordered by (similarity desc, id asc).  The reference returns
 *               HashMap order here, which is unspecified; this is the order the top-k search uses.
 *   rerank = 1: every candidate re-ranked as in the top-k search (sequential dp in the caller's order, a row's last pair of a
 *               dim wins, total_cmp with NaN canonicalised, ties to the smaller id), not truncated.
 * The number of results is known only after scoring, so they come back in a handle the library owns, in host memory:
 * *out receives it (NULL on failure), cdb_sparse_results_offsets gives the number of queries and offsets[n_queries+1]
 * (query q's results are entries [offsets[q], offsets[q+1])), cdb_sparse_results_read copies the entries of queries
 * [first_query, first_query + n_queries) -- offsets[first+n] - offsets[first] of them -- best first, and
 * cdb_sparse_results_destroy frees it (NULL is a no-op).  The handle does not reference the index: appends, deletes and
 * destroying the index afterwards leave it unchanged; reads of one handle are re-entrant.  n_queries = 0 or an index
 * without rows gives a handle of n_queries empty queries without running anything on the device.  Null arguments,
 * malformed query CSR and a read range past the handle's queries are CDB_INVALID_PARAMS, refused before the device is
 * touched.  There is no device-memory form: a caller could not size its result buffers before the call.  Device scratch
 * is bounded by searching the queries in chunks (512 MB of scratch; a chunk holds at least one query); failing
 * allocations are CDB_CUDA_ERROR and leave nothing allocated.  The index's live rows must be fewer than 2^31. */
typedef struct cdb_sparse_results cdb_sparse_results; /* opaque, host memory */
cdb_status cdb_sparse_search_batch_all(cdb_sparse_index *index, const uint64_t *q_offsets, const uint32_t *q_dims,
                                       const float *q_values, uint32_t n_queries, const cdb_sparse_search_params *params,
                                       cdb_sparse_results **out);
cdb_status cdb_sparse_results_offsets(const cdb_sparse_results *results, uint32_t *out_n_queries, uint64_t *out_offsets);
cdb_status cdb_sparse_results_read(const cdb_sparse_results *results, uint32_t first_query, uint32_t n_queries, uint32_t *out_ids,
                                   float *out_scores);
cdb_status cdb_sparse_results_destroy(cdb_sparse_results *results);
/* InvertedIndex::sample_embedding + finalize_sampling (inverted/mod.rs:148-247) over n pair values:
 *   out_counts[t-1] = #values > t for t = 1..9 (prior_counts, may be NULL, added first; prior_values = values they cover)
 *   out_ub = first t with (count as f32 / values as f32) * 100.0 <= clamp_margin_percent, else 10.0 (also with no values) */
cdb_status cdb_sparse_sample_upper_bound(int32_t device, const float *values, uint64_t n, float clamp_margin_percent,
                                         const uint64_t *prior_counts, uint64_t prior_values, uint64_t *out_counts, float *out_ub);
/* the itoe store's live embeddings that have sparse values, in ascending internal-id order (metadata fields are parsed past,
 * raw_vector_embedding.rs:34-64, 91-132).  Host-side readers, no GPU work.
 *   scan -> number of such embeddings, their pairs in total, the largest internal id
 *   load -> entries [first_entry, first_entry + max_entries): internal ids, row_offsets[read+1] (starting at 0), dims and
 *           values (at most max_pairs pairs, else CDB_INVALID_PARAMS)
 *   cdb_sparse_index_append_itoe -> cdb_sparse_index_append of every such embedding; out_internal_ids[r] = the internal id of
 *           appended row r (the first max_ids of them).  The cold start of a collection's sparse index: the caller sets
 *           values_upper_bound to what LMDB holds. */
cdb_status cdb_itoe_scan_sparse(const char *collection_dir, uint64_t *out_entries, uint64_t *out_pairs, uint64_t *out_max_internal_id);
cdb_status cdb_itoe_load_sparse(const char *collection_dir, uint64_t first_entry, uint64_t max_entries, uint64_t max_pairs,
                                uint32_t *out_internal_ids, uint64_t *out_row_offsets, uint32_t *out_dims, float *out_values,
                                uint64_t *out_read);
cdb_status cdb_sparse_index_append_itoe(cdb_sparse_index *index, const char *collection_dir, uint32_t *out_internal_ids,
                                        uint64_t max_ids, uint64_t *out_appended);

/* ------------------------------------------------ TF-IDF / BM25 index
 * TFIDFIndex (src/indexes/tf_idf/mod.rs) over TFIDFIndexRoot (src/models/tf_idf_index.rs) and VersionedVec
 * (src/models/versioned_vec.rs); the search is SparseAnnQueryBasic::search_bm25 (src/models/sparse_ann_query.rs:149-302).
 * Text processing (process_text: tokenize, lowercase, stopwords, stemmer, xxhash32) stays with the caller, which passes
 * what TFIDFIndexRoot::insert receives: per document the (term_hash, tf) pairs, tf = compute_bm25_term_frequency.
 *
 * Documents.  Rows are CSR: row r holds pairs [row_offsets[r], row_offsets[r+1]) and has id id_base + r.  tf is taken as
 * given, 0, -0, negative, inf and NaN included.  A row repeating a hash is CDB_INVALID_PARAMS (process_text never makes
 * one).  counted[r] = 0 marks a row for an id without text (internal ids are shared by a collection's indexes): it must be
 * empty and never counts; counted = NULL counts every row.
 * N (total_documents_count, mod.rs:85-137): +1 per counted row appended, -1 per counted row deleted.
 * df of a term (VersionedVec::len, versioned_vec.rs:131-199): its entries, counted physically -- +1 per row appended with
 * it; a delete in the row's insert version removes the entry (-1); a delete in a later version marks the entry and pushes
 * a tombstone word, both of which count (+1).  So df can exceed N.
 * idf (get_idf, sparse_ann_query.rs:298-302) = log1pf(((N - df) as f32 + 0.5) / (df as f32 + 0.5)) with u32 wrapping
 * N - df and round-to-nearest u32 -> f32, and Rust's f32::ln_1p, the C library's log1pf.  At the end of every append and
 * delete the df of every term is uploaded and the idf computed on the device by the fdlibm log1pf (csrc/bm25_idf.h),
 * which gives glibc's log1pf bits on every non-negative finite float.
 * Versions.  append and delete_rows take the transaction's version; versions passed to either must not decrease (with it
 * every list is in ascending id order, as push_sorted keeps it, versioned_vec.rs:207-226).
 *
 * Score (search_bm25).  A query is a list of term hashes (the query's own tf is not used).  Hashes the index never saw are
 * skipped; a repeated hash counts once per occurrence.  A document's score is its first product tf * idf, then += of the
 * later ones, f32 without FMA and not started from 0 (0 + -0 would turn a -0 score into +0).  The products are added in
 * the caller's query-term order.  The reference adds them in its BinaryHeap's pop order, which is the same for documents
 * that match at most 2 query terms (f32 addition commutes); with more terms the two can differ in the last bits, by at
 * most gamma_{m-1} * (sum of the products) when every product is positive.  A term whose list has no live entry adds
 * nothing; the reference can panic on it (unreachable! in PostingListHead::cmp once such a head meets another).
 * Top-k (search_bm25's 512 buckets).  Document d competes in bucket d % 512 and replaces its holder only if
 * score > bucket score (which starts at -inf): NaN and -inf never enter, equal scores (+0 and -0 too) stay with the smaller
 * id.  The winners are sorted by f32::total_cmp descending (+0 above -0), ties to the smaller id (the reference's
 * sort_unstable leaves ties open), and truncated to k; k = 0 is the reference's top_k None.  out_ids / out_scores have
 * kout = (k == 0 || k > 512) ? 512 : k columns; unused slots hold CDB_INVALID_ID / 0, out_counts[q] = filled slots.
 * Deleted rows are never results.
 *
 * Deviations.  Deleting a deleted row is a no-op (the reference decrements N again).  The reference packs an entry as
 * id << 32 | tf bits and reads every word with bit 63 set as a tombstone, so it never returns an id >= 2^31; here every id
 * below id_base + capacity_rows <= 2^32 - 1 is searched.
 * Searches on one handle are re-entrant; append and delete take the handle exclusively and first wait for the searches
 * already enqueued on the device.  An append that fails changes nothing.  Without a CUDA device every compute entry point
 * returns CDB_CUDA_ERROR. */
typedef struct cdb_tfidf_index cdb_tfidf_index; /* opaque */

typedef struct {
    int32_t device;
    uint64_t capacity_rows;   /* id_base + capacity_rows <= 2^32 - 1 */
    uint64_t capacity_pairs;  /* (term_hash, tf) pairs over all rows */
    uint32_t id_base;
} cdb_tfidf_index_desc;

cdb_status cdb_tfidf_index_create(const cdb_tfidf_index_desc *desc, cdb_tfidf_index **out);
cdb_status cdb_tfidf_index_destroy(cdb_tfidf_index *index);
uint64_t cdb_tfidf_index_size(const cdb_tfidf_index *index);
/* n rows inserted at `version`; row_offsets[n+1] (row_offsets[0] = 0), hashes / tfs [row_offsets[n]], counted [n] or NULL */
cdb_status cdb_tfidf_index_append(cdb_tfidf_index *index, const uint64_t *row_offsets, const uint32_t *hashes, const float *tfs,
                                  const uint8_t *counted, uint64_t n, uint32_t version);
/* deletes rows[0..n) (local rows < cdb_tfidf_index_size) at `version` */
cdb_status cdb_tfidf_index_delete_rows(cdb_tfidf_index *index, const uint32_t *rows, uint64_t n, uint32_t version);
/* out[i] = 1 if row first+i is deleted (first + n <= capacity_rows); *out_total = deleted rows (either may be NULL) */
cdb_status cdb_tfidf_index_deleted_rows(const cdb_tfidf_index *index, uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total);
/* df and the device's idf of hashes[0..n), and N; a hash the index never saw gets df 0 and idf NaN (any may be NULL) */
cdb_status cdb_tfidf_index_term_stats(cdb_tfidf_index *index, const uint32_t *hashes, uint64_t n, uint32_t *out_df, float *out_idf,
                                      uint32_t *out_documents_count);
/* B queries as CSR of hashes (q_offsets[B+1]); out_ids / out_scores [B][kout], out_counts [B] */
cdb_status cdb_tfidf_search_batch(cdb_tfidf_index *index, const uint64_t *q_offsets, const uint32_t *q_hashes, uint32_t n_queries,
                                  uint32_t k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts);
/* same with every array in DEVICE memory on the index's device, asynchronous on `stream` (NULL = the legacy default stream) */
cdb_status cdb_tfidf_search_batch_device(cdb_tfidf_index *index, const uint64_t *d_q_offsets, const uint32_t *d_q_hashes,
                                         uint32_t n_queries, uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                         void *stream);

/* ---- the reference's TF-IDF index files (<collection>/tf_idf_index: index-tree.dim and <version>.idat, written by
 * TFIDFIndexRoot::serialize and the serializers in src/models/serializer/tf_idf), read as TFIDFIndexRoot::deserialize reads them
 * (src/models/tf_idf_index.rs:369-401).  Host-side, no GPU work.  Format and rules: DESIGN.md section 8d.
 *   open   walks the tree (node dims checked against their tree position, child-offset cycles refused), reads every term
 *          slot (a later slot of a quotient replaces an earlier one; hash = quotient << 16 | dim), walks each list's record
 *          chain (offset and version cycles refused; a list without a record of its slot's version refused) and applies
 *          the tombstones.  A missing file, a truncated node or record, an offset past a file's end, a cycle or a wrong dim
 *          is CDB_INVALID_PARAMS with a message.  The files stay mapped until close.
 *   info   info[6] = {N (total_documents_count), terms, list records kept, live words, largest live id + 1 (0 if none),
 *          largest version of a kept record}
 *   read   terms ascending by hash: hashes[terms], df[terms] (VersionedVec::len after deserialize: every word of the kept
 *          records, marked and tombstone words included), offsets[terms + 1] (CSR into the live words, offsets[0] = 0) and
 *          per live word in list order doc_ids, tfs and versions (of the record holding it).  A live word is neither
 *          u64::MAX, nor marked by a tombstone, nor a tombstone (bit 63), so its id is below 2^31.  Any pointer but files
 *          may be NULL. */
typedef struct cdb_tfidf_files cdb_tfidf_files; /* opaque */
cdb_status cdb_tfidf_files_open(const char *tf_idf_index_dir, cdb_tfidf_files **out);
cdb_status cdb_tfidf_files_close(cdb_tfidf_files *files);
cdb_status cdb_tfidf_files_info(const cdb_tfidf_files *files, uint64_t *info);
cdb_status cdb_tfidf_files_read(const cdb_tfidf_files *files, uint32_t *hashes, uint32_t *df, uint64_t *offsets, uint32_t *doc_ids,
                                float *tfs, uint32_t *versions);
/* Loads the files into an EMPTY index (no row, no term, N = 0): the state the reference serves after deserialize, so that
 * searches, term_stats and every later append and delete under the rules above equal the reference's.
 *   rows      row r (id id_base + r, r < n_rows <= capacity_rows) holds the live words whose id is id_base + r, ascending by
 *             hash.  Words of ids outside [id_base, id_base + n_rows) are skipped (another shard's).  A row is counted when
 *             it has a live word or counted[r] = 1 (a document whose text was all stopwords); counted[r] = 0 on a row with a
 *             live word is refused; counted = NULL marks nothing more.  A row's insert version is that of the record
 *             holding its words; a row whose words carry two versions is refused, and so is one repeating a hash.  A row
 *             deleted before the files were written comes back empty and not deleted.  counted must name only live
 *             documents with text: a deleted document's row is not in the tombstone bitmap, so with counted[r] = 1 it
 *             would count, and a later delete of it would lower N again.
 *   stats     carry_stats = 1: N is the files' N and every term of the files is known with its file df.  carry_stats = 0:
 *             N = 0 and the hashes of the loaded rows are known with df 0.  The index's version is the files' largest.
 *   groups    a shard group sums N and df over its shards in wrapping u32, so load exactly one shard of a group with
 *             carry_stats = 1 and the others with 0, each over its own id range: group searches, and later appends and
 *             deletes on any shard, then equal the one index loaded with the stats.  A shard loaded without them serves
 *             only group searches (its own N and df are not the corpus's).
 *   limits    more live pairs for the rows than capacity_pairs (or 2^31 or more) is CDB_INVALID_PARAMS.
 * The device decodes, sorts and scatters the words; the host only copies the records into pinned staging memory (at most
 * 256 MB) and marks the tombstoned positions.  The handle is held exclusively, as by an append, after the searches already
 * enqueued have drained.  A load that fails leaves the index empty and usable. */
cdb_status cdb_tfidf_index_load_files(cdb_tfidf_index *index, const cdb_tfidf_files *files, uint64_t n_rows, const uint8_t *counted,
                                      int32_t carry_stats);

/* ------------------------------------------------ multi-GPU: row-sharded sparse and TF-IDF search
 * The sparse and TF-IDF indexes of a collection split over the slots of a cdb_shard_group, next to (or without) its dense
 * shards: a slot holds at most one dense, one sparse and one TF-IDF shard, and one group and one communicator serve all
 * three.  Each shard is an ordinary index whose id_base is the global id of its local row 0; appends and deletes go to the
 * owning shard (TF-IDF with the same versions the whole index would see).
 * Contract: ids, counts and score bits equal what cdb_sparse_search_batch / cdb_tfidf_search_batch return for ONE index
 * holding every shard's rows at their global ids, with the same appends, deletes and versions.
 *   attach      CDB_INVALID_PARAMS for a shard on another device than its slot and, in a local group
 *               (cdb_shard_group_create), for sparse shards whose quantization_bits or values_upper_bound bits differ from
 *               another slot's, and for shards of one kind whose [id_base, id_base + capacity_rows) ranges overlap.  In a
 *               per-rank group (cdb_shard_group_create_rank) the caller guarantees both across the ranks, as it does id
 *               ranges for dense shards.
 *   search      CDB_INVALID_PARAMS, before any device work, for null arguments, malformed query CSR, a local slot without a
 *               shard of that kind, and the single-index limits: sparse k in 1..1024 and k * f <= 5120; TF-IDF k keeps its
 *               meaning (0 = top_k None, above 512 gives 512 columns).  In a per-rank group every rank calls the search with
 *               the same batch and receives the same result.
 *   sparse      every shard keeps its top m = k * f candidates (f = reranking_factor with rerank, else 1) and one all-gather
 *               brings them to every rank, which selects the group's top m: the single index's candidates, since keys are
 *               unique and each shard's top m holds every one of its rows in the group's top m.  Without rerank these are
 *               the results.  With rerank each rank re-ranks only the candidates it owns, a second all-gather combines them,
 *               and the top k of the m re-ranked keys are kept.  (Re-ranking each shard's own top m and merging would not be
 *               the same: a row outside the group's top m can re-rank into the top k.)  Queries are searched in chunks that
 *               keep the gather buffer within 256 MB; each local shard holds its reader lock through both phases.
 *               The device form (per-rank groups only) takes device arrays and is asynchronous on `stream`.
 *   TF-IDF      idf depends on the whole corpus: N = sum of the shards' N, df = sum of their df (u32, wrapping), and idf
 *               computed with the function a single index uses (csrc/bm25_idf.h).  Both forms run one plan on the device:
 *               each local slot writes its shard's [N, df of every query term], one all-gather of 1 + query terms u32 per
 *               rank brings them to every rank, and a kernel sums them and computes the idf of every query term; the host
 *               never waits in between.  Each shard scores under that idf and hands in all 512 bucket winners per query;
 *               per bucket the best of the ranks wins with `>`, equal scores (+0 and -0 too) going to the smaller id, then
 *               they are sorted and truncated as in cdb_tfidf_search_batch.  Each local shard holds its reader lock from
 *               the df look-up through the scoring. */
cdb_status cdb_shard_group_attach_sparse(cdb_shard_group *group, uint32_t local_slot, cdb_sparse_index *shard);
cdb_status cdb_shard_group_attach_tfidf(cdb_shard_group *group, uint32_t local_slot, cdb_tfidf_index *shard);
cdb_status cdb_sparse_search_batch_sharded(cdb_shard_group *group, const uint64_t *q_offsets, const uint32_t *q_dims,
                                           const float *q_values, uint32_t n_queries, const cdb_sparse_search_params *params,
                                           uint32_t *out_ids, float *out_scores, uint32_t *out_counts);
cdb_status cdb_sparse_search_batch_sharded_device(cdb_shard_group *group, const uint64_t *d_q_offsets, const uint32_t *d_q_dims,
                                                  const float *d_q_values, uint32_t n_queries, const cdb_sparse_search_params *params,
                                                  uint32_t *d_ids, float *d_scores, uint32_t *d_counts, void *stream);
cdb_status cdb_tfidf_search_batch_sharded(cdb_shard_group *group, const uint64_t *q_offsets, const uint32_t *q_hashes, uint32_t n_queries,
                                          uint32_t k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts);
/* The TF-IDF search with every array in DEVICE memory, asynchronous on `stream` (NULL = the legacy default stream): no host
 * synchronisation and no device-to-host copy.  Ids, counts and score bits equal cdb_tfidf_search_batch_sharded's on the same
 * group and batch: it runs the host form's plan, on the caller's stream.  n_query_hashes must equal d_q_offsets[n_queries]
 * (d_q_offsets[0] = 0): the host sizes the df exchange by it.  The device CSR is not validated, but no kernel reads
 * d_q_hashes at or past n_query_hashes.  Served groups: those whose local slots all sit on one device, the one holding the
 * caller's arrays -- per-rank groups, one-slot local groups and loopback groups (a device listed more than once).
 * CDB_INVALID_PARAMS, before any device work: null arguments (with n_queries > 0), n_query_hashes >= 2^31, a local group
 * spanning devices, a local slot without a TF-IDF shard.  n_queries = 0 returns with nothing launched. */
cdb_status cdb_tfidf_search_batch_sharded_device(cdb_shard_group *group, const uint64_t *d_q_offsets, const uint32_t *d_q_hashes,
                                                 uint32_t n_queries, uint64_t n_query_hashes, uint32_t k, uint32_t *d_ids,
                                                 float *d_scores, uint32_t *d_counts, void *stream);
/* Sparse top_k None over the group (params->k = 0): every candidate of every query, in a cdb_sparse_results handle read
 * with cdb_sparse_results_offsets / _read / _destroy.  Contract: offsets, ids and score bits equal what
 * cdb_sparse_search_batch_all returns for ONE index holding every shard's rows at their global ids, with the same appends
 * and deletes, with and without rerank: a row's candidacy and its re-ranked score depend only on the query, the params and
 * the row, and the result order is a total order on unique keys, so each shard scores, re-ranks and sorts its own
 * candidates and the group merges the ranks' sorted runs.
 *   refusals    CDB_INVALID_PARAMS before any device work, in cdb_sparse_search_batch_all's order: null group, params or
 *               out; params->k != 0; malformed query CSR; null query pairs; then a local slot without a sparse shard.
 *               A group whose shards hold 2^31 live rows or more in total is CDB_INVALID_PARAMS on every rank.
 *   exchange    one all-gather of each rank's tiles and live rows (per-rank groups only), then per chunk of queries (the
 *               same chunk on every rank, from the group's largest shard) one all-gather of the per-query candidate counts
 *               and all-gathers of the sorted keys in sub-batches of queries whose gather buffer stays within 256 MB (a
 *               sub-batch holds at least one query).  Local slot 0 merges and copies the results to the host.
 *   n_queries = 0 gives a handle of 0 queries without a collective.  In a per-rank group every rank calls with the same
 *   batch and receives the same handle contents.  Host form only: the result size is known only after scoring.  Each
 *   local shard holds its reader lock until every stream has drained. */
cdb_status cdb_sparse_search_batch_all_sharded(cdb_shard_group *group, const uint64_t *q_offsets, const uint32_t *q_dims,
                                               const float *q_values, uint32_t n_queries, const cdb_sparse_search_params *params,
                                               cdb_sparse_results **out);

/* ------------------------------------------------ hybrid search (reciprocal-rank fusion)
 * hybrid_search (src/api/vectordb/search/repo.rs:168-341) and batch_hybrid_search (repo.rs:343-555); request defaults
 * top_k = 10, fusion_constant_k = 60.0 (src/api/vectordb/search/dtos.rs:6-12).
 *
 * Lists.  A request names two sources, DenseAndSparse, DenseAndTFIDF or SparseAndTFIDF (dtos.rs:73-90), and searches each
 * with top_k Some(3 * top_k): the dense side is hnsw_index.search without a filter, TF-IDF returns at most 512 results (its
 * buckets).  The first list is the one named first: dense before sparse, dense before TF-IDF, sparse before TF-IDF.
 * Score.  The entry at 0-based position rank of a list contributes 1.0 / (rank as f32 + k + f32::EPSILON), f32, left to
 * right, one rounding per operation ((rank + k) + eps and rank + (k + eps) round differently for some small negative k;
 * never at k = 60).  The source's own score is not used.
 * Key.  Entries are keyed by VectorId after remap_search_results (src/indexes/mod.rs:248-258), which is the internal id:
 * a collection's indexes share them.  Dense results of a graph with metadata carry replica ids, which
 * get_raw_emb_by_internal_id (src/models/collection.rs:358-384) maps to id - id % max_replica_per_node, so the replicas of
 * one embedding are one key: id_stride = max_replica_per_node does the same here (0 or 1 = the id itself).
 * Combining (FxHashMap final_scores).  First list: insert, so a key listed twice keeps its worse-ranked occurrence's
 * score.  Second list: the batch form's and_modify(+=).or_insert(score) -- a key not in the first list starts from its
 * first occurrence's score, every later occurrence adds.  Sums are f32 without FMA, in rank order.  The single form's
 * or_insert(0.0).0 += score gives the same result except for a key only in the second list whose score is -0.0 (k = -inf),
 * where 0.0 + -0.0 = +0.0; these entry points compute the batch form.
 * Output.  Every distinct key, sorted by f32::total_cmp descending, ties to the smaller id (the reference's sort_unstable
 * leaves them open).  The reference does NOT truncate to top_k (select_nth_unstable_by only partitions), so a query holds
 * up to the whole union, 6 * top_k entries; a caller that wants top_k truncates.  Unused slots hold CDB_INVALID_ID / 0 and
 * out_counts[q] = distinct keys.
 * k.  Any f32: a negative k only logs a warning in the reference.  A zero denominator gives +inf, k = +inf gives +0 and
 * k = -inf gives -0 scores, k near 3e38 gives subnormal scores (no flush to zero).  A NaN k makes every score NaN with
 * k's payload and the quiet bit set (0xFFA00001 -> 0xFFE00001), as x86 SSE propagates it.  No other NaN or -inf arises.
 * Threshold.  batch_hybrid_search searches the sparse side with early_terminate_threshold None (the config value) where
 * hybrid_search passes the request's; here it is sparse_params.early_terminate_threshold, one value per call -- a single
 * request is a batch of 1.  A batch that mixes kinds of request goes to cdb_hybrid_search_batch_mixed[_sharded][_device]
 * below, which searches each source once for every query that names it. */

/* Generic fusion of two ranked id lists per query: ids [B][ld], counts [B] (entries below min(count, ld) are taken as
 * given, CDB_INVALID_ID included), id_stride per list as above.  out_ids / out_scores [B][ld_out], out_counts [B].
 * ld_first + ld_second > 2048 or ld_out < ld_first + ld_second: CDB_INVALID_PARAMS, checked before the device is touched.
 * Use it for lists this library did not produce in one call: sharded dense results merged per query, or the replica-id
 * results of cdb_search_batch_filtered (id_stride = max_replica_per_node). */
cdb_status cdb_rrf_fuse(int32_t device, const uint32_t *first_ids, const uint32_t *first_counts, uint32_t ld_first,
                        uint32_t first_id_stride, const uint32_t *second_ids, const uint32_t *second_counts, uint32_t ld_second,
                        uint32_t second_id_stride, uint32_t n_queries, float fusion_constant_k, uint32_t ld_out, uint32_t *out_ids,
                        float *out_scores, uint32_t *out_counts);
/* same with every array in DEVICE memory on `device`, asynchronous on `stream` (NULL = the legacy default stream) */
cdb_status cdb_rrf_fuse_device(int32_t device, const uint32_t *d_first_ids, const uint32_t *d_first_counts, uint32_t ld_first,
                               uint32_t first_id_stride, const uint32_t *d_second_ids, const uint32_t *d_second_counts,
                               uint32_t ld_second, uint32_t second_id_stride, uint32_t n_queries, float fusion_constant_k,
                               uint32_t ld_out, uint32_t *d_out_ids, float *d_out_scores, uint32_t *d_out_counts, void *stream);

/* The two sources of a composed hybrid search: exactly two of the three handles are set (the third is NULL).  Queries are
 * host arrays for cdb_hybrid_search_batch and device arrays for cdb_hybrid_search_batch_device.  The k of each params
 * struct is ignored: every sub-search runs with k = 3 * top_k (TF-IDF: min(3 * top_k, 512) results). */
typedef struct {
    cdb_index *dense;
    const float *dense_queries;               /* [B][dim] raw f32 */
    cdb_search_params dense_params;           /* mode, ef_search, shortlist_size, ... of cdb_search_batch */
    cdb_sparse_index *sparse;
    const uint64_t *sparse_offsets;           /* CSR [B+1] */
    const uint32_t *sparse_dims;
    const float *sparse_values;
    cdb_sparse_search_params sparse_params;
    cdb_tfidf_index *tfidf;
    const uint64_t *tfidf_offsets;            /* CSR [B+1] of term hashes */
    const uint32_t *tfidf_hashes;
} cdb_hybrid_sources;

/* Composed hybrid search: the batch of one kind of cdb_hybrid_search_batch_mixed[_device] (below) in which every query
 * names the two given sources.  Both sub-searches run through their public *_search_batch_device entry points, the second
 * on a side stream forked from and joined back to the caller's stream (the device form's `stream`; NULL = the legacy
 * default stream) so the two overlap, then one fusion on the caller's stream; intermediate lists live in stream-ordered
 * scratch, and no stream, event or allocation outlives the call's work.
 * out_ids / out_scores [B][6 * top_k], out_counts [B]; err_flags [B] (may be NULL) receives the dense search's flags and
 * is written only when a dense source is given.
 * Each sub-search takes its own handle's shared lock and sees that handle as of its own enqueue; there is no snapshot
 * across the two handles (the reference takes none either).  Appends and deletes keep their contracts: they wait for the
 * searches already enqueued on the device.
 * CDB_INVALID_PARAMS: null sources or a source count other than two, then the refusals of the mixed form: top_k > 341 (the
 * dense and sparse searches take k <= 1024), CDB_SEARCH_ALL_CANDIDATES, null queries, a sparse source with rerank and
 * 3 * top_k * reranking_factor > 5120, malformed host query CSR, handles on different devices.
 * CDB_UNSUPPORTED: a dense handle with graph metadata (its HNSW searches go through cdb_search_batch_filtered[_device];
 * attach it to a one-slot shard group and use cdb_hybrid_search_batch_sharded, below).  Refusals of a sub-search's own parameter
 * checks are returned as that search returns them.  B = 0 or top_k = 0: empty results (out_counts zeroed), no kernel
 * launched. */
cdb_status cdb_hybrid_search_batch(const cdb_hybrid_sources *sources, uint32_t n_queries, uint32_t top_k, float fusion_constant_k,
                                   uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags);
cdb_status cdb_hybrid_search_batch_device(const cdb_hybrid_sources *sources, uint32_t n_queries, uint32_t top_k,
                                          float fusion_constant_k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                          uint8_t *d_err_flags, void *stream);

/* Hybrid search over a shard group (DESIGN.md section 8h): the group's dense, sparse and TF-IDF shards are already
 * attached, so the sources name kinds, not handles; exactly two of use_dense, use_sparse, use_tfidf are 1.  The k of each
 * params struct is ignored, as above.  dense_id_stride is the first list's id_stride when the dense side is first:
 * max_replica_per_node for replica graphs, 0 or 1 when ids are keys; every other list has stride 1. */
typedef struct {
    uint32_t use_dense, use_sparse, use_tfidf;
    const float *dense_queries;               /* [B][dim] raw f32 */
    cdb_search_params dense_params;
    uint32_t dense_id_stride;
    const uint64_t *sparse_offsets;           /* CSR [B+1] */
    const uint32_t *sparse_dims;
    const float *sparse_values;
    cdb_sparse_search_params sparse_params;
    const uint64_t *tfidf_offsets;            /* CSR [B+1] of term hashes */
    const uint32_t *tfidf_hashes;
} cdb_hybrid_group_sources;

/* The group's two sub-searches at k = 3 * top_k, as cdb_search_batch_sharded / cdb_search_batch_filtered_sharded,
 * cdb_sparse_search_batch_sharded and cdb_tfidf_search_batch_sharded return them, fused on the device with the contract
 * above (lists, scores, keys, output [B][6 * top_k], err_flags written only with a dense source and OR-ed over the ranks).
 * Dense side: when every local dense shard has graph metadata, the filtered path with no filter on any query (the
 * reference's hnsw_index.search(.., None) for a collection with a metadata schema; results carry replica ids, so pass
 * dense_id_stride = max_replica_per_node); when none has, the path of cdb_search_batch_sharded in any mode.  A group of
 * one local slot (cdb_shard_group_create with one device) is a real group, so a single index with graph metadata gets its
 * hybrid search here, which cdb_hybrid_search_batch refuses.
 * The call is the batch of one kind of cdb_hybrid_search_batch_mixed_sharded[_device] (below) in which every query names
 * the two given sources.  Both sub-searches run under one hold of the group's lock, one after the other in list order on
 * the group's streams (the caller's stream in the device form), so every rank issues the same collectives in the same
 * order; the first list lives in scratch of this call until the fusion on local slot 0 (this rank's device in a per-rank
 * group), which every rank runs and so ends with the same rows.  Queries are fused in chunks that keep both intermediate
 * lists within 256 MB.  The host form copies nothing back but the fused ids, scores, counts and error bytes.
 * CDB_INVALID_PARAMS, before any copy or launch: null sources or a source count other than two, then the refusals of the
 * mixed form: a null output or group; top_k > 341; CDB_SEARCH_ALL_CANDIDATES in dense_params; null queries of a named
 * source; sparse rerank with 3 * top_k * reranking_factor > 5120; malformed query CSR (host form); the sparse search's
 * other parameter checks; a local slot without a shard of a named kind; local dense shards of which some have graph
 * metadata and some do not, or a mode other than CDB_MODE_HNSW on metadata shards; world * 3 * top_k * 8 > 200 KB (the
 * dense merge).  B = 0 or top_k = 0: counts zeroed, nothing launched.
 * The device form serves groups of one local slot (per-rank groups and one-device local groups), takes device arrays and
 * is asynchronous on `stream` (NULL = the legacy default stream): its work follows what `stream` held, and the caller's
 * later work on `stream` follows it.  It refuses a TF-IDF source with CDB_UNSUPPORTED, before the group is read: the host
 * sizes the TF-IDF idf exchange by the batch's term count, and cdb_hybrid_group_sources carries none. */
cdb_status cdb_hybrid_search_batch_sharded(cdb_shard_group *group, const cdb_hybrid_group_sources *sources, uint32_t n_queries,
                                           uint32_t top_k, float fusion_constant_k, uint32_t *out_ids, float *out_scores,
                                           uint32_t *out_counts, uint8_t *err_flags);
cdb_status cdb_hybrid_search_batch_sharded_device(cdb_shard_group *group, const cdb_hybrid_group_sources *sources,
                                                  uint32_t n_queries, uint32_t top_k, float fusion_constant_k, uint32_t *d_ids,
                                                  float *d_scores, uint32_t *d_counts, uint8_t *d_err_flags, void *stream);

/* ------------------------------------------------ hybrid search over mixed batches
 * batch_hybrid_search (repo.rs:343-555) takes a batch in which each query names its own pair of sources.  kinds[q] is
 * query q's pair: the first list is the source the kind names first. */
enum { CDB_HYBRID_DENSE_SPARSE = 0, CDB_HYBRID_DENSE_TFIDF = 1, CDB_HYBRID_SPARSE_TFIDF = 2 };

/* A mixed batch of B queries.  kinds [B] is HOST memory in both forms (request metadata, read to plan the call).  A source's
 * queries are those whose kind names it, in request order (the reference's dense_queries, sparse_queries and
 * tfidf_queries): n_dense = the DENSE_SPARSE and DENSE_TFIDF queries, n_sparse = the DENSE_SPARSE and SPARSE_TFIDF ones,
 * n_tfidf = the DENSE_TFIDF and SPARSE_TFIDF ones (host counts).  A source with a count of 0 is not searched and its
 * handle and queries may be NULL.  Queries are host arrays for cdb_hybrid_search_batch_mixed and device arrays for the
 * device form; the k of each params struct is ignored, as above. */
typedef struct {
    const uint8_t *kinds;                     /* [B] CDB_HYBRID_*, host memory */
    uint32_t n_dense, n_sparse, n_tfidf;
    cdb_index *dense;
    const float *dense_queries;               /* [n_dense][dim] raw f32 */
    cdb_search_params dense_params;
    cdb_sparse_index *sparse;
    const uint64_t *sparse_offsets;           /* CSR [n_sparse + 1] */
    const uint32_t *sparse_dims;
    const float *sparse_values;
    cdb_sparse_search_params sparse_params;
    cdb_tfidf_index *tfidf;
    const uint64_t *tfidf_offsets;            /* CSR [n_tfidf + 1] of term hashes */
    const uint32_t *tfidf_hashes;
} cdb_hybrid_mixed_sources;

/* Hybrid search over a mixed batch (DESIGN.md section 8i).  Row q is, bit for bit in ids, counts and score bits, the row
 * cdb_hybrid_search_batch returns for query q when the batch is split by kind (queries are independent): every source
 * with queries is searched ONCE, at k = 3 * top_k (TF-IDF: min(3 * top_k, 512) results), the first on the caller's stream
 * and the others on side streams forked from and joined back to it, then each kind present is fused with one launch
 * straight into its queries' rows.  out_ids / out_scores [B][6 * top_k], out_counts [B]; err_flags [B] (may be NULL)
 * receives the dense search's flags of each query that names the dense source and 0 for SPARSE_TFIDF queries.
 * sparse_params is one value per call: the batch form passes early_terminate_threshold None (the config value) and
 * ignores the per-query thresholds, as the reference does.  Locks and snapshots as cdb_hybrid_search_batch.
 * CDB_INVALID_PARAMS, before any copy or launch: null sources or output; top_k > 341; null kinds with B > 0; a kind above 2;
 * counts that disagree with kinds; CDB_SEARCH_ALL_CANDIDATES with dense queries; a null handle or null queries of a source
 * with queries; sparse rerank with 3 * top_k * reranking_factor > 5120; malformed host query CSR (host form); handles of
 * the searched sources on different devices.  CDB_UNSUPPORTED: a dense handle with graph metadata (use a one-slot shard
 * group and cdb_hybrid_search_batch_mixed_sharded).  B = 0 or top_k = 0: counts zeroed, no kernel launched. */
cdb_status cdb_hybrid_search_batch_mixed(const cdb_hybrid_mixed_sources *sources, uint32_t n_queries, uint32_t top_k,
                                         float fusion_constant_k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts,
                                         uint8_t *err_flags);
cdb_status cdb_hybrid_search_batch_mixed_device(const cdb_hybrid_mixed_sources *sources, uint32_t n_queries, uint32_t top_k,
                                                float fusion_constant_k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts,
                                                uint8_t *d_err_flags, void *stream);

/* A mixed batch over a shard group: the fields of cdb_hybrid_mixed_sources with the group's shards in place of handles (a
 * source with queries needs a shard of its kind in every local slot).  dense_id_stride is the dense list's id_stride, as in
 * cdb_hybrid_group_sources.  n_tfidf_hashes is the term count of the TF-IDF CSR (tfidf_offsets[n_tfidf]): the device form
 * sizes the group's idf exchange by it (the host form reads it from the offsets and ignores the field). */
typedef struct {
    const uint8_t *kinds;                     /* [B] CDB_HYBRID_*, host memory */
    uint32_t n_dense, n_sparse, n_tfidf;
    const float *dense_queries;               /* [n_dense][dim] raw f32 */
    cdb_search_params dense_params;
    uint32_t dense_id_stride;
    const uint64_t *sparse_offsets;           /* CSR [n_sparse + 1] */
    const uint32_t *sparse_dims;
    const float *sparse_values;
    cdb_sparse_search_params sparse_params;
    const uint64_t *tfidf_offsets;            /* CSR [n_tfidf + 1] of term hashes */
    const uint32_t *tfidf_hashes;
    uint64_t n_tfidf_hashes;
} cdb_hybrid_group_mixed_sources;

/* The contract of cdb_hybrid_search_batch_mixed over the group: row q is the row cdb_hybrid_search_batch_sharded returns
 * for query q when the batch is split by kind, and err_flags are OR-ed over the ranks.  Under one hold of the group's lock
 * the sources with queries run one after the other in the order dense, sparse, TF-IDF; a source without queries issues no
 * collective.  Every rank passes the same kinds, so every rank issues the same collectives.  The TF-IDF idf step runs once
 * per call over the TF-IDF queries.  Request positions are taken in chunks that keep the intermediate lists within 256 MB;
 * a chunk is one contiguous range of each source's queries, each sub-search takes its range and the fusion the chunk.
 * The host form stages each source's queries once per local device.  The device form serves groups of one local slot and
 * takes device arrays, TF-IDF included, asynchronously on `stream` (NULL = the legacy default stream).
 * CDB_INVALID_PARAMS, before any copy or launch: the refusals of cdb_hybrid_search_batch_mixed that need no handle, n_tfidf_hashes
 * >= 2^31, then under the group's lock those of cdb_hybrid_search_batch_sharded: a local slot without a shard of a searched
 * kind, local dense shards of which some have graph metadata and some do not (or a mode other than CDB_MODE_HNSW on
 * metadata shards), world * 3 * top_k * 8 > 200 KB (the dense merge).  B = 0 or top_k = 0: counts zeroed, nothing launched. */
cdb_status cdb_hybrid_search_batch_mixed_sharded(cdb_shard_group *group, const cdb_hybrid_group_mixed_sources *sources,
                                                 uint32_t n_queries, uint32_t top_k, float fusion_constant_k, uint32_t *out_ids,
                                                 float *out_scores, uint32_t *out_counts, uint8_t *err_flags);
cdb_status cdb_hybrid_search_batch_mixed_sharded_device(cdb_shard_group *group, const cdb_hybrid_group_mixed_sources *sources,
                                                        uint32_t n_queries, uint32_t top_k, float fusion_constant_k, uint32_t *d_ids,
                                                        float *d_scores, uint32_t *d_counts, uint8_t *d_err_flags, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* COSDATA_B200_H */
