"""CPU-side checks of hybrid search over mixed batches (cdb_hybrid_search_batch_mixed[_sharded][_device]):
  * tests/pyhybrid_mixed.fuse_mixed against a literal restatement of batch_hybrid_search's query_mapping loop, and against the
    batch split by kind, each part fused with fuse_batch and the rows put back in request order;
  * every refusal that comes before a handle or the group is read, on stand-in handles and a stand-in group pointing at
    zeroed memory, in all four entry points;
  * the bindings: ctypes prototypes and structs, the C++ mirror, INTEGRATION.md's extern block and Rust structs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from tests import pyhybrid as ph
from tests import pyhybrid_mixed as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INV = cdb.Status.INVALID_PARAMS
ENTRIES = ("cdb_hybrid_search_batch_mixed", "cdb_hybrid_search_batch_mixed_device", "cdb_hybrid_search_batch_mixed_sharded",
           "cdb_hybrid_search_batch_mixed_sharded_device")


def last_error():
    return (_lib.load().cdb_last_error_string() or b"").decode()


# ---------------------------------------------------------------- the Python restatement
def source_lists(rng, kinds, ld, id_range=40):
    """random ranked lists for each source's batch (duplicates and short counts included)"""
    _, n = pm.query_mapping(kinds)
    out = {}
    for name, rows in n.items():
        if rows:
            ids = rng.integers(0, id_range, size=(rows, ld[name])).astype(np.uint32)
            out[name] = (ids, rng.integers(0, ld[name] + 3, size=rows).astype(np.uint32))
    return out


def literal_mixed(kinds, lists, k, ld_out):
    """repo.rs:343-555 written out: the mapping built while the batches are, then each query's two lists by name"""
    mapping, n_d, n_s, n_t = [], 0, 0, 0
    for q, kind in enumerate(kinds):
        if kind == 0:
            mapping.append((q, n_d, n_s, "dense_sparse")); n_d += 1; n_s += 1
        elif kind == 1:
            mapping.append((q, n_d, n_t, "dense_tfidf")); n_d += 1; n_t += 1
        else:
            mapping.append((q, n_s, n_t, "sparse_tfidf")); n_s += 1; n_t += 1
    ids = np.full((len(kinds), ld_out), 0xFFFFFFFF, np.uint32)
    scores = np.zeros((len(kinds), ld_out), np.float32)
    counts = np.zeros(len(kinds), np.uint32)
    for q, i1, i2, kind in mapping:
        first, second = {"dense_sparse": ("dense", "sparse"), "dense_tfidf": ("dense", "tfidf"), "sparse_tfidf": ("sparse", "tfidf")}[kind]
        a, ca = lists[first]
        b, cb = lists[second]
        r = ph.fuse(a[i1, :min(int(ca[i1]), a.shape[1])].tolist(), b[i2, :min(int(cb[i2]), b.shape[1])].tolist(), k)
        counts[q] = len(r)
        for j, (key, s) in enumerate(r):
            ids[q, j], scores[q, j] = key, s
    return ids, scores, counts


def split_by_kind(kinds, lists, k, ld_out):
    """what a caller without the mixed entry point does: one fuse_batch per kind, rows put back in request order"""
    mapping, _ = pm.query_mapping(kinds)
    ids = np.zeros((len(kinds), ld_out), np.uint32)
    scores = np.zeros((len(kinds), ld_out), np.float32)
    counts = np.zeros(len(kinds), np.uint32)
    for kind, (first, second) in enumerate(pm.KIND_SOURCES):
        mine = [m for m in mapping if m[3] == kind]
        if not mine:
            continue
        q, i1, i2 = (np.array([m[j] for m in mine]) for j in range(3))
        a, ca = lists[first]
        b, cb = lists[second]
        r = ph.fuse_batch(a[i1], ca[i1], b[i2], cb[i2], k, ld_out=ld_out)
        ids[q], scores[q], counts[q] = r
    return ids, scores, counts


@pytest.mark.parametrize("seed", range(6))
def test_fuse_mixed_equals_the_literal_loop_and_the_split_by_kind(seed):
    rng = np.random.default_rng(seed)
    nq = [1, 7, 30, 64, 5, 40][seed]
    kinds = rng.integers(0, 3, nq).astype(np.uint8) if seed != 4 else np.full(nq, 2, np.uint8)
    ld = {"dense": 6, "sparse": 6, "tfidf": 4}
    lists = source_lists(rng, kinds, ld)
    k = [60.0, 1.0, -3.5, 60.0, 0.5, 1e3][seed]
    ld_out = 12
    got = pm.fuse_mixed(kinds, lists, k, ld_out=ld_out)
    for want in (literal_mixed(kinds, lists, k, ld_out), split_by_kind(kinds, lists, k, ld_out)):
        assert np.array_equal(got[2], want[2])
        for q in range(nq):
            c = int(got[2][q])
            assert np.array_equal(got[0][q, :c], want[0][q, :c])
            assert np.array_equal(got[1][q, :c].view(np.uint32), want[1][q, :c].view(np.uint32))


def test_query_mapping_counts_each_source():
    mapping, n = pm.query_mapping([0, 2, 1, 1, 0, 2])
    assert n == {"dense": 4, "sparse": 4, "tfidf": 4}
    assert mapping == [(0, 0, 0, 0), (1, 1, 0, 2), (2, 1, 1, 1), (3, 2, 2, 1), (4, 3, 2, 0), (5, 3, 3, 2)]


def test_split_mixed_builds_each_source_batch_in_request_order():
    kinds = [2, 0, 1]
    dense = np.arange(6, dtype=np.float32).reshape(3, 2)
    sparse = [[(1, 1.0)], [(2, 2.0)], None]
    tfidf = [[7], None, [9, 10]]
    k, b = cdb.split_mixed(kinds, dense, sparse, tfidf)
    assert k.dtype == np.uint8 and k.tolist() == kinds
    assert np.array_equal(b["dense"], dense[[1, 2]])
    assert b["sparse"] == [[(1, 1.0)], [(2, 2.0)]] and b["tfidf"] == [[7], [9, 10]]
    _, b = cdb.split_mixed([2, 2], None, [[], []], [[1], [2]])
    assert set(b) == {"sparse", "tfidf"}
    with pytest.raises(ValueError):
        cdb.split_mixed([0], None, [[]], None)
    with pytest.raises(ValueError):
        cdb.split_mixed([3], None, None, None)


# ---------------------------------------------------------------- refusals before any handle or group is read
class Call:
    """one request of B = 3 queries of kinds [0, 1, 2] (two queries for each source) on stand-in handles and group"""

    def __init__(self):
        self.blob = (C.c_uint8 * 4096)()
        self.handle = C.cast(self.blob, C.c_void_p)
        self.kinds = np.array([0, 1, 2], np.uint8)
        self.q = np.zeros(64, np.float32)
        self.off = np.array([0, 1, 2], np.uint64)
        self.bad_off = np.array([0, 2, 1], np.uint64)
        self.dims = np.zeros(2, np.uint32)
        self.vals = np.zeros(2, np.float32)
        self.out = np.zeros(8192, np.uint32)
        self.cnt = np.zeros(4, np.uint32)

    def fill(self, s, counts=(2, 2, 2), rerank=0, factor=5, all_candidates=False, null=None, bad_csr=None, kinds=None):
        s.kinds = (self.kinds if kinds is None else kinds).ctypes.data
        s.n_dense, s.n_sparse, s.n_tfidf = counts
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

    def single(self, **kw):
        s = _lib.HybridMixedSources()
        s.dense = s.sparse = s.tfidf = self.handle
        return self.fill(s, **kw)

    def group_src(self, **kw):
        s = _lib.HybridGroupMixedSources()
        s.n_tfidf_hashes = 2
        return self.fill(s, **kw)

    def run(self, form, src, nq=3, top_k=10, out=True):
        L = _lib.load()
        o = self.out.ctypes.data if out else None
        c = self.cnt.ctypes.data if out else None
        p = C.byref(src) if src is not None else None
        if form == "host":
            return L.cdb_hybrid_search_batch_mixed(p, nq, top_k, 60.0, o, o, c, None)
        if form == "device":
            return L.cdb_hybrid_search_batch_mixed_device(p, nq, top_k, 60.0, o, o, c, None, None)
        if form == "group":
            return L.cdb_hybrid_search_batch_mixed_sharded(self.handle, p, nq, top_k, 60.0, o, o, c, None)
        return L.cdb_hybrid_search_batch_mixed_sharded_device(self.handle, p, nq, top_k, 60.0, o, o, c, None, None)

    def src(self, form, **kw):
        return self.single(**kw) if form in ("host", "device") else self.group_src(**kw)


FORMS = ("host", "device", "group", "group_device")


@pytest.mark.parametrize("form", FORMS)
def test_refusals_come_before_any_handle_or_group_is_read(form):
    c = Call()
    assert c.run(form, None) == INV and "null sources" in last_error()
    assert c.run(form, c.src(form), out=False) == INV and "null output" in last_error()
    assert c.run(form, c.src(form), top_k=342) == INV and "341" in last_error()
    assert c.run(form, c.src(form, null="kinds")) == INV and "null kinds" in last_error()
    assert c.run(form, c.src(form, kinds=np.array([0, 3, 2], np.uint8))) == INV and "kinds[1] = 3" in last_error()
    for counts in ((2, 2, 1), (3, 2, 2), (2, 1, 2), (0, 0, 0)):
        assert c.run(form, c.src(form, counts=counts)) == INV and "n_dense, n_sparse and n_tfidf" in last_error()
    assert c.run(form, c.src(form), nq=2) == INV and "n_dense, n_sparse and n_tfidf" in last_error()
    assert c.run(form, c.src(form, all_candidates=True)) == INV and "CDB_SEARCH_ALL_CANDIDATES" in last_error()
    nulls = ["dense_queries", "sparse_offsets", "tfidf_offsets"] + (["dense", "sparse", "tfidf"] if form in ("host", "device") else [])
    for null in nulls:
        assert c.run(form, c.src(form, null=null)) == INV and "null" in last_error()
    assert c.run(form, c.src(form, rerank=1, factor=6), top_k=341) == INV and "reranking_factor" in last_error()
    assert c.run(form, c.src(form, rerank=1, factor=0)) == INV and "reranking_factor" in last_error()
    if form in ("host", "group"):
        # the host forms read the query CSRs
        for bad in ("sparse", "tfidf"):
            assert c.run(form, c.src(form, bad_csr=bad)) == INV and "offsets" in last_error()
        assert c.run(form, c.src(form, null="sparse_dims")) == INV and "null sparse query pairs" in last_error()
        assert c.run(form, c.src(form, null="tfidf_hashes")) == INV and "null tf-idf query hashes" in last_error()


def test_a_source_without_queries_is_not_read():
    """sparse + TF-IDF queries only: the dense handle and queries are null and its params would be refused, yet the
    refusal names the next thing wrong (a null sparse handle; the stand-in group's missing slot)"""
    c = Call()
    kinds = np.array([2, 2, 2], np.uint8)
    s = c.single(counts=(0, 3, 3), kinds=kinds, null="dense_queries", all_candidates=True)
    s.dense = s.sparse = None
    assert c.run("device", s) == INV and "null sparse handle" in last_error()
    s = c.group_src(counts=(0, 3, 3), kinds=kinds, null="dense_queries", all_candidates=True)
    assert c.run("group_device", s) == INV and "one local slot" in last_error()


def test_an_empty_batch_needs_no_kinds_and_no_device():
    c = Call()
    for form in ("host", "device"):
        s = c.single(counts=(0, 0, 0), null="kinds")
        s.dense = s.sparse = s.tfidf = None
        assert c.run(form, s, nq=0, out=False) == 0, last_error()


def test_kind_constants():
    hdr = open(os.path.join(ROOT, "include", "cosdata_b200.h")).read()
    enum = re.search(r"enum \{ CDB_HYBRID_DENSE_SPARSE = 0, CDB_HYBRID_DENSE_TFIDF = 1, CDB_HYBRID_SPARSE_TFIDF = 2 \};", hdr)
    assert enum
    assert (_lib.HYBRID_DENSE_SPARSE, _lib.HYBRID_DENSE_TFIDF, _lib.HYBRID_SPARSE_TFIDF) == (0, 1, 2)
    assert pm.KIND_SOURCES == cdb.api.HYBRID_KIND_SOURCES


# ---------------------------------------------------------------- bindings
def struct_fields(hdr, name):
    body = hdr[:hdr.index("} %s;" % name)]
    body = body[body.rindex("typedef struct {") + len("typedef struct {"):]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(\w+)\s*(?:,|;)", body)


def test_bindings_agree():
    lib = _lib.load()
    structs = {"cdb_hybrid_search_batch_mixed": _lib.HybridMixedSources, "cdb_hybrid_search_batch_mixed_device": _lib.HybridMixedSources,
               "cdb_hybrid_search_batch_mixed_sharded": _lib.HybridGroupMixedSources,
               "cdb_hybrid_search_batch_mixed_sharded_device": _lib.HybridGroupMixedSources}
    hdr = open(os.path.join(ROOT, "include", "cosdata_b200.h")).read()
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    hpp = open(os.path.join(ROOT, "include", "cosdata_b200.hpp")).read()
    for name in ENTRIES:
        assert hasattr(lib, name) and name in _lib.PROTOTYPES
        args = _lib.PROTOTYPES[name][1]
        assert args[1 if "sharded" in name else 0]._type_ is structs[name]
        assert re.search(rf"\b{name}\s*\(", hdr) and f"pub fn {name}(" in doc
    assert "cdb_hybrid_search_batch_mixed_sharded(" in hpp and "hybrid_search_mixed(" in hpp
    for cname, cls in (("cdb_hybrid_mixed_sources", _lib.HybridMixedSources), ("cdb_hybrid_group_mixed_sources", _lib.HybridGroupMixedSources)):
        fields = struct_fields(hdr, cname)
        assert fields == [f for f, _ in cls._fields_]
        rust = re.search(rf"pub struct {cname} \{{(.*?)\n\}}", doc, re.S).group(1)
        assert re.findall(r"pub (\w+):", rust) == fields
