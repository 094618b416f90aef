"""cosdata_b200 -- H100-native (sm_90a) implementation of cosdata's ANN distance hot path.

The package is a thin host mirror of the reference's operator surface over the
C ABI in include/cosdata_b200.h; all compute lives in csrc/*.cu.
"""
from .api import (  # noqa: F401
    INVALID_ID, CosdataError, DenseIndex, HnswFiles, DistanceError, DistanceMetric, DistanceMetricKind,
    ScalarQuantization, SearchMode, Status, Storage, StorageType, code_bytes, debug_set_hnsw_flags, device_count,
    itoe_get, itoe_load, itoe_scan, kernel_launch_count, prop_file_load, prop_file_load_metadata, prop_file_scan, sample_values_range, sample_values_range_device, synth_matrix, tensor_peak,
    SparseIndex, SparseResults, SparseSearchOptions, itoe_load_sparse, itoe_scan_sparse, sparse_csr, sparse_sample_upper_bound,
    TfIdfFiles, TfIdfIndex, average_document_length, bm25_term_frequency, debug_bm25_device, debug_bm25_host,
    hybrid_batch_search, hybrid_batch_search_mixed, hybrid_sources, rrf_fuse, split_mixed,
)
