"""ctypes loader for libcosdata_b200.so -- the only way Python reaches the kernels.

There is no fallback: if the shared object is missing or a symbol declared in
include/cosdata_b200.h is absent, import-time use fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcosdata_b200.so")

c_u8p = C.c_void_p
c_f32p = C.c_void_p
c_u32p = C.c_void_p
c_i32p = C.c_void_p
c_vp = C.c_void_p


class IndexDesc(C.Structure):
    _fields_ = [
        ("dim", C.c_uint32),
        ("storage_type", C.c_int32),
        ("metric", C.c_int32),
        ("range_lo", C.c_float),
        ("range_hi", C.c_float),
        ("capacity", C.c_uint64),
        ("device", C.c_int32),
        ("keep_raw_f32", C.c_int32),
        ("id_base", C.c_uint32),
        ("tensor_prefilter", C.c_uint32),
    ]


class GraphDesc(C.Structure):
    _fields_ = [
        ("num_levels", C.c_uint32),
        ("neighbors_count", C.c_uint32),
        ("level0_neighbors_count", C.c_uint32),
        ("entry", C.c_uint32),
        ("root_row", C.c_uint32),
        ("level_counts", C.c_void_p),
        ("node_row", C.c_void_p),
        ("adjacency", C.c_void_p),
        ("child", C.c_void_p),
    ]


class GraphMetadata(C.Structure):
    _fields_ = [
        ("md_dims", C.c_uint32),
        ("n_md", C.c_uint32),
        ("md_bits", C.c_void_p),
        ("md_mags", C.c_void_p),
        ("node_id", C.c_void_p),
        ("node_md", C.c_void_p),
        ("pseudo_entry", C.c_uint32),
    ]


class VectorDataBatch(C.Structure):
    _fields_ = [
        ("codes", C.c_void_p),
        ("mags", C.c_void_p),
        ("ids", C.c_void_p),
        ("has_id", C.c_void_p),
        ("md_bits", C.c_void_p),
        ("md_mags", C.c_void_p),
        ("has_md", C.c_void_p),
    ]


class BuildParams(C.Structure):
    _fields_ = [
        ("num_levels", C.c_uint32),
        ("neighbors_count", C.c_uint32),
        ("level0_neighbors_count", C.c_uint32),
        ("ef_construction", C.c_uint32),
        ("shortlist_size", C.c_uint32),
        ("max_batch", C.c_uint32),
        ("seed", C.c_uint64),
    ]


class ReplicaBuild(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint32),
        ("row", C.c_void_p), ("node_id", C.c_void_p), ("base_id", C.c_void_p), ("md_row", C.c_void_p), ("max_level", C.c_void_p),
        ("md_dims", C.c_uint32), ("n_md", C.c_uint32),
        ("md_bits", C.c_void_p), ("md_mags", C.c_void_p),
        ("main_root_md", C.c_uint32), ("pseudo_root_md", C.c_uint32),
    ]


class ReplicaInsert(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint32),
        ("row", C.c_void_p), ("node_id", C.c_void_p), ("base_id", C.c_void_p), ("md_row", C.c_void_p), ("max_level", C.c_void_p),
        ("md_dims", C.c_uint32), ("n_md_new", C.c_uint32),
        ("md_bits_new", C.c_void_p), ("md_mags_new", C.c_void_p),
    ]


class SearchParams(C.Structure):
    _fields_ = [
        ("k", C.c_uint32),
        ("mode", C.c_int32),
        ("ef_search", C.c_uint32),
        ("shortlist_size", C.c_uint32),
        ("exact_only", C.c_int32),
        ("prefilter_k", C.c_uint32),
        ("flags", C.c_uint32),            # CDB_SEARCH_* bits
        ("reserved1", C.c_uint32),
    ]


class SparseIndexDesc(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("quantization_bits", C.c_uint32),
        ("values_upper_bound", C.c_float),
        ("capacity_rows", C.c_uint64),
        ("capacity_pairs", C.c_uint64),
        ("id_base", C.c_uint32),
    ]


class SparseSearchParams(C.Structure):
    _fields_ = [
        ("k", C.c_uint32),
        ("early_terminate_threshold", C.c_float),
        ("rerank", C.c_int32),
        ("reranking_factor", C.c_uint32),
    ]


class TfIdfIndexDesc(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("capacity_rows", C.c_uint64),
        ("capacity_pairs", C.c_uint64),
        ("id_base", C.c_uint32),
    ]


class HybridSources(C.Structure):
    _fields_ = [
        ("dense", C.c_void_p),
        ("dense_queries", C.c_void_p),
        ("dense_params", SearchParams),
        ("sparse", C.c_void_p),
        ("sparse_offsets", C.c_void_p),
        ("sparse_dims", C.c_void_p),
        ("sparse_values", C.c_void_p),
        ("sparse_params", SparseSearchParams),
        ("tfidf", C.c_void_p),
        ("tfidf_offsets", C.c_void_p),
        ("tfidf_hashes", C.c_void_p),
    ]


class HybridGroupSources(C.Structure):
    _fields_ = [
        ("use_dense", C.c_uint32),
        ("use_sparse", C.c_uint32),
        ("use_tfidf", C.c_uint32),
        ("dense_queries", C.c_void_p),
        ("dense_params", SearchParams),
        ("dense_id_stride", C.c_uint32),
        ("sparse_offsets", C.c_void_p),
        ("sparse_dims", C.c_void_p),
        ("sparse_values", C.c_void_p),
        ("sparse_params", SparseSearchParams),
        ("tfidf_offsets", C.c_void_p),
        ("tfidf_hashes", C.c_void_p),
    ]


HYBRID_DENSE_SPARSE, HYBRID_DENSE_TFIDF, HYBRID_SPARSE_TFIDF = 0, 1, 2   # CDB_HYBRID_*: a mixed batch's kinds


class HybridMixedSources(C.Structure):
    _fields_ = [
        ("kinds", C.c_void_p),
        ("n_dense", C.c_uint32),
        ("n_sparse", C.c_uint32),
        ("n_tfidf", C.c_uint32),
        ("dense", C.c_void_p),
        ("dense_queries", C.c_void_p),
        ("dense_params", SearchParams),
        ("sparse", C.c_void_p),
        ("sparse_offsets", C.c_void_p),
        ("sparse_dims", C.c_void_p),
        ("sparse_values", C.c_void_p),
        ("sparse_params", SparseSearchParams),
        ("tfidf", C.c_void_p),
        ("tfidf_offsets", C.c_void_p),
        ("tfidf_hashes", C.c_void_p),
    ]


class HybridGroupMixedSources(C.Structure):
    _fields_ = [
        ("kinds", C.c_void_p),
        ("n_dense", C.c_uint32),
        ("n_sparse", C.c_uint32),
        ("n_tfidf", C.c_uint32),
        ("dense_queries", C.c_void_p),
        ("dense_params", SearchParams),
        ("dense_id_stride", C.c_uint32),
        ("sparse_offsets", C.c_void_p),
        ("sparse_dims", C.c_void_p),
        ("sparse_values", C.c_void_p),
        ("sparse_params", SparseSearchParams),
        ("tfidf_offsets", C.c_void_p),
        ("tfidf_hashes", C.c_void_p),
        ("n_tfidf_hashes", C.c_uint64),
    ]


# symbol -> (restype, argtypes); must list every function of include/cosdata_b200.h
PROTOTYPES = {
    "cdb_abi_version": (C.c_int32, []),
    "cdb_last_error_string": (C.c_char_p, []),
    "cdb_device_count": (C.c_int32, [C.POINTER(C.c_int32)]),
    "cdb_synth_fill_host": (C.c_int32, [C.c_uint64, C.c_uint64, C.c_uint64, c_f32p]),
    "cdb_code_bytes": (C.c_size_t, [C.c_int32, C.c_uint32]),
    "cdb_sample_values_range": (C.c_int32, [C.c_int32, c_f32p, C.c_uint64, C.c_uint32, C.c_float, c_vp, C.c_uint64, c_vp, c_f32p]),
    "cdb_sample_values_range_device": (C.c_int32, [C.c_int32, c_vp, C.c_uint64, C.c_uint32, C.c_float, c_vp, C.c_uint64, c_vp, c_f32p, c_vp]),
    "cdb_index_describe": (C.c_int32, [c_vp, c_vp]),
    "cdb_prop_file_scan": (C.c_int32, [C.c_char_p, c_vp, c_vp, c_vp, c_vp]),
    "cdb_prop_file_load": (C.c_int32, [C.c_char_p, C.c_uint64, C.c_uint64, c_vp, c_vp, c_f32p, c_vp, c_vp, c_vp]),
    "cdb_index_append_prop_file": (C.c_int32, [c_vp, C.c_char_p, c_vp, C.c_uint64, c_vp]),
    "cdb_itoe_scan": (C.c_int32, [C.c_char_p, c_vp, c_vp, c_vp]),
    "cdb_itoe_load": (C.c_int32, [C.c_char_p, C.c_uint64, C.c_uint64, c_vp, c_f32p, c_vp]),
    "cdb_itoe_get": (C.c_int32, [C.c_char_p, C.c_uint32, c_f32p, C.c_uint32, c_vp]),
    "cdb_index_append_itoe": (C.c_int32, [c_vp, C.c_char_p, c_vp, C.c_uint64, c_vp]),
    "cdb_distance_pairs_md": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, c_vp, c_vp, C.c_uint64, c_f32p, c_vp]),
    "cdb_index_set_graph_metadata": (C.c_int32, [c_vp, c_vp]),
    "cdb_search_batch_filtered": (C.c_int32, [c_vp, c_f32p, C.c_uint32, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32p, c_vp, c_vp]),
    "cdb_prop_file_scan_metadata": (C.c_int32, [C.c_char_p, c_vp, c_vp]),
    "cdb_prop_file_load_metadata": (C.c_int32, [C.c_char_p, C.c_uint64, C.c_uint32, c_vp, c_f32p, c_vp, c_vp, c_vp, c_vp]),
    "cdb_hnsw_files_open": (C.c_int32, [C.c_char_p, C.c_uint32, C.c_uint32, c_vp]),
    "cdb_hnsw_files_open_versioned": (C.c_int32, [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, c_vp]),
    "cdb_hnsw_files_close": (C.c_int32, [c_vp]),
    "cdb_hnsw_files_info": (C.c_int32, [c_vp, c_vp, c_vp]),
    "cdb_hnsw_files_level": (C.c_int32, [c_vp, C.c_uint32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "cdb_hnsw_files_metadata": (C.c_int32, [c_vp, c_vp, c_f32p]),
    "cdb_hnsw_files_slot_scores": (C.c_int32, [c_vp, C.c_uint32, c_vp, c_vp]),
    "cdb_index_set_graph_slot_scores": (C.c_int32, [C.c_void_p, c_vp, c_vp]),
    "cdb_index_set_graph_from_files": (C.c_int32, [c_vp, c_vp]),
    "cdb_quantize_batch": (C.c_int32, [C.c_int32, C.c_int32, C.c_float, C.c_float, c_f32p, C.c_uint64, C.c_uint32, c_vp, c_f32p]),
    "cdb_distance_pairs": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_uint32, c_vp, c_f32p, c_vp, c_f32p, C.c_uint64, c_f32p, c_i32p]),
    "cdb_index_create": (C.c_int32, [C.POINTER(IndexDesc), C.POINTER(C.c_void_p)]),
    "cdb_index_destroy": (C.c_int32, [C.c_void_p]),
    "cdb_index_size": (C.c_uint64, [C.c_void_p]),
    "cdb_index_append_f32": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint64]),
    "cdb_index_append_f32_device": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "cdb_index_append_codes": (C.c_int32, [C.c_void_p, c_vp, c_f32p, C.c_uint64]),
    "cdb_index_append_synthetic": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]),
    "cdb_index_read_codes": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, c_vp, c_f32p]),
    "cdb_index_set_graph": (C.c_int32, [C.c_void_p, C.POINTER(GraphDesc)]),
    "cdb_index_build_graph": (C.c_int32, [C.c_void_p, C.POINTER(BuildParams)]),
    "cdb_index_build_graph_replicas": (C.c_int32, [C.c_void_p, C.POINTER(BuildParams), C.POINTER(ReplicaBuild), C.c_void_p]),
    "cdb_index_read_graph_metadata_level": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "cdb_index_graph_info": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "cdb_index_read_graph_level": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cdb_index_insert_graph": (C.c_int32, [C.c_void_p, C.POINTER(BuildParams), c_vp, c_vp, C.POINTER(C.c_uint64)]),
    "cdb_index_insert_graph_replicas": (C.c_int32, [C.c_void_p, C.POINTER(BuildParams), C.POINTER(ReplicaInsert), c_vp,
                                                    C.POINTER(C.c_uint64)]),
    "cdb_index_read_graph_slot_scores": (C.c_int32, [C.c_void_p, C.c_uint32, c_vp]),
    "cdb_index_delete_rows": (C.c_int32, [C.c_void_p, c_vp, C.c_uint64, C.c_uint32, C.c_uint32, c_vp, C.POINTER(C.c_uint64)]),
    "cdb_index_delete_rows_replicas": (C.c_int32, [C.c_void_p, c_vp, C.c_uint64, C.c_uint32, C.c_uint32, c_vp, C.POINTER(C.c_uint64)]),
    "cdb_index_read_replica_slot_scores": (C.c_int32, [C.c_void_p, C.c_uint32, c_vp]),
    "cdb_index_deleted_rows": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, c_vp, C.POINTER(C.c_uint64)]),
    "cdb_index_hnsw_counters": (C.c_int32, [C.c_void_p, C.c_void_p]),
    "cdb_search_batch": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint32, C.POINTER(SearchParams), c_u32p, c_f32p, c_u32p, c_u8p]),
    "cdb_search_batch_device": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint32, C.POINTER(SearchParams), c_u32p, c_f32p, c_u32p, c_u8p, C.c_void_p]),
    "cdb_search_batch_filtered_device": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint32, C.POINTER(SearchParams), c_u32p, c_vp, C.c_uint32,
                                                     c_u8p, c_u32p, c_f32p, c_u32p, c_u8p, C.c_void_p]),
    "cdb_score_ids": (C.c_int32, [C.c_void_p, c_f32p, c_u32p, C.c_uint32, c_f32p, c_i32p]),
    "cdb_rerank_f32": (C.c_int32, [C.c_void_p, c_f32p, c_u32p, C.c_uint32, C.c_uint32, c_u32p, c_f32p, c_u32p]),
    "cdb_nccl_unique_id": (C.c_int32, [C.c_void_p]),
    "cdb_shard_group_create": (C.c_int32, [C.c_void_p, C.c_uint32, c_vp]),
    "cdb_shard_group_create_rank": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int32, c_vp]),
    "cdb_shard_group_destroy": (C.c_int32, [C.c_void_p]),
    "cdb_shard_group_attach": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "cdb_shard_group_world": (C.c_uint32, [C.c_void_p]),
    "cdb_search_batch_sharded": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cdb_search_batch_sharded_device": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cdb_search_batch_filtered_sharded": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint32, C.POINTER(SearchParams), c_u32p, c_vp, c_u8p, c_u32p,
                                                      c_f32p, c_u32p, c_u8p]),
    "cdb_search_batch_filtered_sharded_device": (C.c_int32, [C.c_void_p, c_f32p, C.c_uint32, C.POINTER(SearchParams), c_u32p, c_vp,
                                                             C.c_uint32, c_u8p, c_u32p, c_f32p, c_u32p, c_u8p, C.c_void_p]),
    "cdb_shard_group_attach_sparse": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "cdb_shard_group_attach_tfidf": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "cdb_sparse_search_batch_sharded": (C.c_int32, [C.c_void_p, c_vp, c_vp, c_vp, C.c_uint32, C.POINTER(SparseSearchParams), c_vp, c_vp, c_vp]),
    "cdb_sparse_search_batch_sharded_device": (C.c_int32, [C.c_void_p, c_vp, c_vp, c_vp, C.c_uint32, C.POINTER(SparseSearchParams), c_vp,
                                                           c_vp, c_vp, C.c_void_p]),
    "cdb_sparse_search_batch_all_sharded": (C.c_int32, [C.c_void_p, c_vp, c_vp, c_vp, C.c_uint32, C.POINTER(SparseSearchParams),
                                                        C.POINTER(C.c_void_p)]),
    "cdb_tfidf_search_batch_sharded": (C.c_int32, [C.c_void_p, c_vp, c_vp, C.c_uint32, C.c_uint32, c_vp, c_vp, c_vp]),
    "cdb_tfidf_search_batch_sharded_device": (C.c_int32, [C.c_void_p, c_vp, c_vp, C.c_uint32, C.c_uint64, C.c_uint32, c_vp, c_vp, c_vp,
                                                          C.c_void_p]),
    "cdb_merge_topk_device": (C.c_int32, [C.c_int32, C.c_int32, c_u32p, c_f32p, C.c_uint32, C.c_uint32, C.c_uint32, c_u32p, c_f32p, C.c_void_p]),
    "cdb_kernel_launch_count": (C.c_uint64, []),
    "cdb_index_last_kernel_ms": (C.c_int32, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "cdb_index_hnsw_profile": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "cdb_debug_set_hnsw_flags": (C.c_int32, [C.c_uint32]),
    "cdb_debug_tensor_peak": (C.c_int32, [C.c_int32, C.c_int32, C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_float)]),
    "cdb_debug_bm25": (C.c_int32, [C.c_int32, c_f32p, C.c_uint64, c_f32p, c_u32p, c_u32p, C.c_uint64, c_f32p, C.c_void_p]),
    "cdb_index_set_raw_f32": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]),
    "cdb_index_raw_missing": (C.c_uint64, [C.c_void_p]),
    "cdb_index_fill_raw_from_itoe": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "cdb_index_stats": (C.c_int32, [C.c_void_p, C.c_void_p]),
    "cdb_index_stats_ex": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32]),
    "cdb_index_last_candidate_counts": (C.c_int32, [C.c_void_p, C.c_uint32, c_u32p]),
    "cdb_index_scan_ms_history": (C.c_int32, [C.c_void_p, C.c_uint32, c_f32p, C.POINTER(C.c_uint32)]),
    "cdb_sparse_index_create": (C.c_int32, [C.POINTER(SparseIndexDesc), C.POINTER(C.c_void_p)]),
    "cdb_sparse_index_destroy": (C.c_int32, [C.c_void_p]),
    "cdb_sparse_index_size": (C.c_uint64, [C.c_void_p]),
    "cdb_sparse_index_append": (C.c_int32, [C.c_void_p, c_vp, c_u32p, c_f32p, C.c_uint64]),
    "cdb_sparse_index_delete_rows": (C.c_int32, [C.c_void_p, c_u32p, C.c_uint64]),
    "cdb_sparse_index_deleted_rows": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, c_u8p, C.POINTER(C.c_uint64)]),
    "cdb_sparse_search_batch": (C.c_int32, [C.c_void_p, c_vp, c_u32p, c_f32p, C.c_uint32, C.POINTER(SparseSearchParams),
                                            c_u32p, c_f32p, c_u32p]),
    "cdb_sparse_search_batch_device": (C.c_int32, [C.c_void_p, c_vp, c_u32p, c_f32p, C.c_uint32, C.POINTER(SparseSearchParams),
                                                   c_u32p, c_f32p, c_u32p, C.c_void_p]),
    "cdb_sparse_search_batch_all": (C.c_int32, [C.c_void_p, c_vp, c_u32p, c_f32p, C.c_uint32, C.POINTER(SparseSearchParams),
                                                C.POINTER(C.c_void_p)]),
    "cdb_sparse_results_offsets": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32), c_vp]),
    "cdb_sparse_results_read": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, c_u32p, c_f32p]),
    "cdb_sparse_results_destroy": (C.c_int32, [C.c_void_p]),
    "cdb_sparse_sample_upper_bound": (C.c_int32, [C.c_int32, c_f32p, C.c_uint64, C.c_float, c_vp, C.c_uint64, c_vp,
                                                  C.POINTER(C.c_float)]),
    "cdb_itoe_scan_sparse": (C.c_int32, [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "cdb_itoe_load_sparse": (C.c_int32, [C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64, c_u32p, c_vp, c_u32p, c_f32p,
                                         C.POINTER(C.c_uint64)]),
    "cdb_sparse_index_append_itoe": (C.c_int32, [C.c_void_p, C.c_char_p, c_u32p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "cdb_tfidf_index_create": (C.c_int32, [C.POINTER(TfIdfIndexDesc), C.POINTER(C.c_void_p)]),
    "cdb_tfidf_index_destroy": (C.c_int32, [C.c_void_p]),
    "cdb_tfidf_index_size": (C.c_uint64, [C.c_void_p]),
    "cdb_tfidf_index_append": (C.c_int32, [C.c_void_p, c_vp, c_u32p, c_f32p, c_u8p, C.c_uint64, C.c_uint32]),
    "cdb_tfidf_index_delete_rows": (C.c_int32, [C.c_void_p, c_u32p, C.c_uint64, C.c_uint32]),
    "cdb_tfidf_index_deleted_rows": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, c_u8p, C.POINTER(C.c_uint64)]),
    "cdb_tfidf_index_term_stats": (C.c_int32, [C.c_void_p, c_u32p, C.c_uint64, c_u32p, c_f32p, C.POINTER(C.c_uint32)]),
    "cdb_tfidf_search_batch": (C.c_int32, [C.c_void_p, c_vp, c_u32p, C.c_uint32, C.c_uint32, c_u32p, c_f32p, c_u32p]),
    "cdb_tfidf_search_batch_device": (C.c_int32, [C.c_void_p, c_vp, c_u32p, C.c_uint32, C.c_uint32, c_u32p, c_f32p, c_u32p,
                                                  C.c_void_p]),
    "cdb_tfidf_files_open": (C.c_int32, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "cdb_tfidf_files_close": (C.c_int32, [C.c_void_p]),
    "cdb_tfidf_files_info": (C.c_int32, [C.c_void_p, c_vp]),
    "cdb_tfidf_files_read": (C.c_int32, [C.c_void_p, c_u32p, c_u32p, c_vp, c_u32p, c_f32p, c_u32p]),
    "cdb_tfidf_index_load_files": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, c_u8p, C.c_int32]),
    "cdb_rrf_fuse": (C.c_int32, [C.c_int32, c_u32p, c_u32p, C.c_uint32, C.c_uint32, c_u32p, c_u32p, C.c_uint32, C.c_uint32,
                                 C.c_uint32, C.c_float, C.c_uint32, c_u32p, c_f32p, c_u32p]),
    "cdb_rrf_fuse_device": (C.c_int32, [C.c_int32, c_u32p, c_u32p, C.c_uint32, C.c_uint32, c_u32p, c_u32p, C.c_uint32,
                                        C.c_uint32, C.c_uint32, C.c_float, C.c_uint32, c_u32p, c_f32p, c_u32p, C.c_void_p]),
    "cdb_hybrid_search_batch": (C.c_int32, [C.POINTER(HybridSources), C.c_uint32, C.c_uint32, C.c_float, c_u32p, c_f32p, c_u32p,
                                            c_u8p]),
    "cdb_hybrid_search_batch_device": (C.c_int32, [C.POINTER(HybridSources), C.c_uint32, C.c_uint32, C.c_float, c_u32p, c_f32p,
                                                   c_u32p, c_u8p, C.c_void_p]),
    "cdb_hybrid_search_batch_sharded": (C.c_int32, [C.c_void_p, C.POINTER(HybridGroupSources), C.c_uint32, C.c_uint32, C.c_float, c_vp,
                                                    c_vp, c_vp, c_vp]),
    "cdb_hybrid_search_batch_sharded_device": (C.c_int32, [C.c_void_p, C.POINTER(HybridGroupSources), C.c_uint32, C.c_uint32, C.c_float,
                                                           c_vp, c_vp, c_vp, c_vp, C.c_void_p]),
    "cdb_hybrid_search_batch_mixed": (C.c_int32, [C.POINTER(HybridMixedSources), C.c_uint32, C.c_uint32, C.c_float, c_u32p, c_f32p,
                                                  c_u32p, c_u8p]),
    "cdb_hybrid_search_batch_mixed_device": (C.c_int32, [C.POINTER(HybridMixedSources), C.c_uint32, C.c_uint32, C.c_float, c_u32p,
                                                         c_f32p, c_u32p, c_u8p, C.c_void_p]),
    "cdb_hybrid_search_batch_mixed_sharded": (C.c_int32, [C.c_void_p, C.POINTER(HybridGroupMixedSources), C.c_uint32, C.c_uint32,
                                                          C.c_float, c_vp, c_vp, c_vp, c_vp]),
    "cdb_hybrid_search_batch_mixed_sharded_device": (C.c_int32, [C.c_void_p, C.POINTER(HybridGroupMixedSources), C.c_uint32,
                                                                 C.c_uint32, C.c_float, c_vp, c_vp, c_vp, c_vp, C.c_void_p]),
}

_lib = None


def load():
    """Load the shared object and bind every declared symbol (raises if anything is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: run `python -m cosdata_b200.build` (nvcc, sm_90a). "
            "There is no CPU fallback for this path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.cdb_abi_version() != 1:
        raise RuntimeError("libcosdata_b200 ABI version mismatch")
    _lib = lib
    return lib
