"""CPU-side checks of cdb_search_batch_filtered_device: the ctypes prototype and INTEGRATION.md's binding exist, and the
argument refusals happen on the host before the handle or the device is touched."""
import ctypes as C
import os
import re

import cosdata_b200 as cdb
from cosdata_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "cdb_search_batch_filtered_device"


def test_prototype_and_binding():
    assert NAME in _lib.PROTOTYPES and len(_lib.PROTOTYPES[NAME][1]) == 13
    assert hasattr(_lib.load(), NAME)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert re.search(r"pub fn " + NAME + r"\(", doc)
    hdr = open(os.path.join(ROOT, "include", "cosdata_b200.h")).read()
    assert re.search(r"CDB_ERRFLAG_BAD_FILTER = 8", hdr)


def test_refusals_before_any_device_work():
    L = _lib.load()
    inv = cdb.Status.INVALID_PARAMS
    ok = _lib.SearchParams(10, int(cdb.SearchMode.HNSW), 64, 64, 0, 0, 0, 0)
    fake = C.c_void_p(16)                                               # device addresses are never dereferenced on the host

    def call(p, offs=fake, dims=fake, n_rows=1, has=fake, ix=None):
        rc = L.cdb_search_batch_filtered_device(ix, fake, 4, None if p is None else C.byref(p), offs, dims, n_rows, has, fake,
                                                fake, fake, fake, None)
        return rc, L.cdb_last_error_string().decode()

    assert call(None) == (inv, "null params")
    bad_mode = _lib.SearchParams(10, int(cdb.SearchMode.BRUTE_RAW), 64, 64, 0, 0, 0, 0)
    assert call(bad_mode) == (inv, "metadata filters apply to CDB_MODE_HNSW")
    for k in (0, 1025):
        assert call(_lib.SearchParams(k, int(cdb.SearchMode.HNSW), 64, 64, 0, 0, 0, 0)) == (inv, "k must be in 1..1024")
    assert call(ok, offs=None) == (inv, "has_filter needs filter_offsets")
    assert call(ok, dims=None, n_rows=3) == (inv, "n_filter_rows > 0 needs filter_dims")
    assert call(ok) == (inv, "null argument")                          # every argument fine but the handle
    assert call(ok, offs=None, has=None, dims=None, n_rows=0) == (inv, "null argument")
