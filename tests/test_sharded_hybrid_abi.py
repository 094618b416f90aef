"""CPU-side checks of the hybrid search over a shard group (cdb_hybrid_search_batch_sharded[_device]): every refusal that
comes before the group is read, on a stand-in group pointing at zeroed memory, and the bindings (ctypes prototypes, the
C++ mirror, INTEGRATION.md's extern block and struct)."""
import ctypes as C
import os
import re

import numpy as np

import cosdata_b200 as cdb
from cosdata_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INV, UNSUP = cdb.Status.INVALID_PARAMS, cdb.Status.UNSUPPORTED
ENTRIES = ("cdb_hybrid_search_batch_sharded", "cdb_hybrid_search_batch_sharded_device")


def last_error():
    return (_lib.load().cdb_last_error_string() or b"").decode()


class Call:
    """one request against a stand-in group; `use` names the sources, the rest adjusts them"""

    def __init__(self):
        self.blob = (C.c_uint8 * 4096)()
        self.group = C.cast(self.blob, C.c_void_p)
        self.q = np.zeros(64, np.float32)
        self.off = np.array([0, 1], np.uint64)
        self.bad_off = np.array([0, 2, 1], np.uint64)
        self.dims = np.zeros(2, np.uint32)
        self.vals = np.zeros(2, np.float32)
        self.out = np.zeros(4096, np.uint32)
        self.cnt = np.zeros(2, np.uint32)

    def sources(self, use, rerank=0, factor=5, all_candidates=False, null=None, bad_csr=None):
        s = _lib.HybridGroupSources()
        s.use_dense, s.use_sparse, s.use_tfidf = ("dense" in use), ("sparse" in use), ("tfidf" in use)
        s.dense_queries = self.q.ctypes.data
        s.dense_params.mode = cdb.SearchMode.HNSW
        s.dense_params.flags = 2 if all_candidates else 0
        off = lambda name: (self.bad_off if bad_csr == name else self.off).ctypes.data   # noqa: E731
        s.sparse_offsets, s.sparse_dims, s.sparse_values = off("sparse"), self.dims.ctypes.data, self.vals.ctypes.data
        s.sparse_params.rerank, s.sparse_params.reranking_factor = rerank, factor
        s.tfidf_offsets, s.tfidf_hashes = off("tfidf"), self.dims.ctypes.data
        if null:
            setattr(s, null, None)
        return s

    def host(self, src, top_k=10, nq=1, group=True, out=True):
        o = self.out.ctypes.data if out else None
        return _lib.load().cdb_hybrid_search_batch_sharded(self.group if group else None, C.byref(src) if src is not None else None, nq,
                                                           top_k, 60.0, o, o, self.cnt.ctypes.data if out else None, None)

    def device(self, src, top_k=10, nq=1, group=True, out=True):
        o = self.out.ctypes.data if out else None
        return _lib.load().cdb_hybrid_search_batch_sharded_device(self.group if group else None,
                                                                  C.byref(src) if src is not None else None, nq, top_k, 60.0, o, o,
                                                                  self.cnt.ctypes.data if out else None, None, None)


def test_refusals_come_before_the_group_is_read():
    c = Call()
    ok = ("sparse", "tfidf")
    for form in (c.host, c.device):
        assert form(c.sources(ok), group=False) == INV and "null group" in last_error()
        assert form(None) == INV and "null sources" in last_error()
        assert form(c.sources(ok), out=False) == INV and "null output" in last_error()
        for use in (("sparse",), ("dense", "sparse", "tfidf"), ()):
            assert form(c.sources(use)) == INV and "exactly two sources" in last_error()
        assert form(c.sources(("dense", "sparse")), top_k=342) == INV and "341" in last_error()
        assert form(c.sources(("dense", "sparse"), rerank=1, factor=6), top_k=341) == INV and "reranking_factor" in last_error()
        assert form(c.sources(("dense", "sparse"), rerank=1, factor=0)) == INV and "reranking_factor" in last_error()
        assert form(c.sources(("dense", "sparse"), all_candidates=True)) == INV and "CDB_SEARCH_ALL_CANDIDATES" in last_error()
        for use, null in ((("dense", "sparse"), "dense_queries"), (("dense", "sparse"), "sparse_offsets"),
                          (("dense", "tfidf"), "tfidf_offsets")):
            assert form(c.sources(use, null=null)) == INV and "null" in last_error()
    # the host form reads the query CSRs
    for use, bad in ((("dense", "sparse"), "sparse"), (("sparse", "tfidf"), "tfidf"), (("dense", "tfidf"), "tfidf")):
        assert c.host(c.sources(use, bad_csr=bad), nq=2) == INV and "offsets" in last_error()
    assert c.host(c.sources(("dense", "sparse"), null="sparse_dims")) == INV and "null sparse query pairs" in last_error()
    assert c.host(c.sources(("sparse", "tfidf"), null="tfidf_hashes")) == INV and "null tf-idf query hashes" in last_error()


def test_device_form_refuses_tfidf_before_the_group_is_read():
    c = Call()
    for use in (("dense", "tfidf"), ("sparse", "tfidf")):
        assert c.device(c.sources(use)) == UNSUP and "host" in last_error()
    # a request it serves is refused only for the stand-in group's missing slot
    assert c.device(c.sources(("dense", "sparse"))) == INV and "one local slot" in last_error()


def test_bindings_agree():
    lib = _lib.load()
    for name in ENTRIES:
        assert hasattr(lib, name) and name in _lib.PROTOTYPES
        assert _lib.PROTOTYPES[name][1][1]._type_ is _lib.HybridGroupSources
    hdr = open(os.path.join(ROOT, "include", "cosdata_b200.h")).read()
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    hpp = open(os.path.join(ROOT, "include", "cosdata_b200.hpp")).read()
    for name in ENTRIES:
        assert re.search(rf"\b{name}\s*\(", hdr) and f"pub fn {name}(" in doc
    assert "cdb_hybrid_search_batch_sharded(" in hpp
    # the struct's fields in the header's order, in ctypes and in the Rust mirror
    body = hdr[:hdr.index("} cdb_hybrid_group_sources;")]
    body = body[body.rindex("typedef struct {") + len("typedef struct {"):]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*(?:,|;)", body)
    assert fields == [f for f, _ in _lib.HybridGroupSources._fields_]
    rust = re.search(r"pub struct cdb_hybrid_group_sources \{(.*?)\n\}", doc, re.S).group(1)
    assert re.findall(r"pub (\w+):", rust) == fields
