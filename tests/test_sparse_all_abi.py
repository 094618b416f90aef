"""CPU-side checks of the top_k None sparse search (cdb_sparse_search_batch_all) and its result handle: refusals happen before
any device work, and without a CUDA device there is no index to search and no CPU fallback."""
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib


def test_refusals_before_touching_the_device():
    L = _lib.load()
    inv = cdb.Status.INVALID_PARAMS
    p = cdb.SparseSearchOptions(None).params()
    assert p.k == 0
    out = C.c_void_p(1)
    qo = np.array([0, 1], np.uint64)
    qd = np.array([1], np.uint32)
    qv = np.array([1.0], np.float32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert L.cdb_sparse_search_batch_all(None, ptr(qo), ptr(qd), ptr(qv), 1, C.byref(p), C.byref(out)) == inv
    assert L.cdb_sparse_results_offsets(None, None, None) == inv
    n = C.c_uint32(0)
    assert L.cdb_sparse_results_offsets(None, C.byref(n), None) == inv
    assert L.cdb_sparse_results_read(None, 0, 0, None, None) == inv
    assert L.cdb_sparse_results_destroy(None) == cdb.Status.OK


def test_no_cpu_fallback_without_device():
    if cdb.device_count() > 0:
        pytest.skip("CUDA device present")
    with pytest.raises(cdb.CosdataError) as e:
        cdb.SparseIndex(capacity_rows=10, capacity_pairs=10).batch_search_all([[(1, 1.0)]], cdb.SparseSearchOptions(None))
    assert e.value.status == cdb.Status.CUDA_ERROR
