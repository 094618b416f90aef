"""CPU-side checks of the sharded TF-IDF search from device buffers (cdb_tfidf_search_batch_sharded_device): the symbol,
its ctypes prototype against the header, the Python binding, and every refusal that comes before the group is read, on
a stand-in group pointing at zeroed memory."""
import ctypes as C
import os
import re

import numpy as np

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import ShardGroup

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "cdb_tfidf_search_batch_sharded_device"
INV = cdb.Status.INVALID_PARAMS


def last_error():
    return (_lib.load().cdb_last_error_string() or b"").decode()


def test_symbol_and_prototype():
    lib = _lib.load()
    assert hasattr(lib, NAME)
    restype, args = _lib.PROTOTYPES[NAME]
    assert restype is C.c_int32
    with open(os.path.join(ROOT, "include", "cosdata_b200.h")) as f:
        hdr = f.read()
    m = re.search(r"cdb_status\s+" + NAME + r"\(([^;]*)\);", hdr)
    assert m, "not declared in the header"
    params = [p.strip() for p in m.group(1).split(",")]
    assert len(params) == len(args) == 10
    # the two host integers between the pointers: n_queries (u32) and n_query_hashes (u64), then k (u32)
    assert params[3].startswith("uint32_t") and args[3] is C.c_uint32
    assert params[4].startswith("uint64_t") and args[4] is C.c_uint64
    assert params[5].startswith("uint32_t") and args[5] is C.c_uint32
    assert hasattr(ShardGroup, "search_tfidf_device")


def test_refusals_before_the_group_is_read():
    lib = _lib.load()
    blob = (C.c_uint8 * 4096)()
    g = C.cast(blob, C.c_void_p)
    buf = np.zeros(64, np.uint64)
    p = buf.ctypes.data

    def call(group=g, off=p, hashes=p, nq=1, nh=1, k=10, ids=p, scores=p, counts=p):
        return lib.cdb_tfidf_search_batch_sharded_device(group, off, hashes, nq, nh, k, ids, scores, counts, None)

    assert call(group=None) == INV and "null argument" in last_error()
    for name in ("off", "ids", "scores", "counts"):
        assert call(**{name: None}) == INV and "null argument" in last_error()
    assert call(hashes=None) == INV and "null query hashes" in last_error()
    assert call(nh=1 << 31) == INV and "2^31" in last_error()
    assert call(nh=(1 << 31) + 5, hashes=None, off=None) == INV and "null argument" in last_error()   # the null check first
    assert call(group=None, nq=0, off=None, ids=None, scores=None, counts=None) == INV and "null argument" in last_error()
