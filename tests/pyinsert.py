"""ctypes binding of tests/hnsw_insert_oracle.c (TEST INFRASTRUCTURE ONLY): the CPU restatement of index_embeddings on a
live graph whose root may sit between data rows.  The shared object is compiled on first use into a temporary directory
(keyed by the sources' contents) and links the checker library oracle/libcosdata_oracle.so."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "hnsw_insert_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    po.lib()   # builds oracle/libcosdata_oracle.so if needed
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_ORACLE, "hnsw_build_internal.h"), os.path.join(_ORACLE, "cosdata_oracle.h")):
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), f"cdb_insert_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-std=gnu11", "-I", _ORACLE,
                        "-o", tmp, _SRC, "-L", _ORACLE, "-lcosdata_oracle", f"-Wl,-rpath,{_ORACLE}", "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, u32, u64, f32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float
    L.ig_init.restype = vp
    L.ig_init.argtypes = [C.c_int, C.c_int, C.c_size_t, u32, u32, u32, u32, u32]
    L.ig_set_table.argtypes = [vp, vp, vp]
    L.ig_insert_rows.argtypes = [vp, u32, u32, vp, u64, u32, u32, vp]
    L.ig_from_graph.restype = vp
    L.ig_from_graph.argtypes = [C.c_int, C.c_int, C.c_size_t, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, vp]
    L.ig_level_count.restype = u32
    L.ig_level_count.argtypes = [vp, u32]
    L.ig_entry.restype = u32
    L.ig_entry.argtypes = [vp]
    L.ig_level_export.argtypes = [vp, u32] + [vp] * 6
    L.ig_search_batch.argtypes = [vp, vp, vp, C.c_size_t, f32, f32, u32, u32, C.c_size_t, vp, vp, vp, vp,
                                  C.POINTER(u64), C.POINTER(u64)]
    L.ig_free.argtypes = [vp]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Graph:
    """A live graph over a growing code table (codes / mags hold every row the graph names; the root is row root_row)."""

    def __init__(self, handle, metric, st, dim, num_levels, nbrs, nbrs0, root_row, codes, mags):
        self.h, self.metric, self.st, self.dim = handle, int(metric), int(st), int(dim)
        self.num_levels, self.nbrs, self.nbrs0, self.root_row = int(num_levels), int(nbrs), int(nbrs0), int(root_row)
        self.set_table(codes, mags)

    def set_table(self, codes, mags):
        self.codes = np.ascontiguousarray(codes, dtype=np.uint8)
        self.mags = np.ascontiguousarray(mags, dtype=np.float32)
        lib().ig_set_table(self.h, _p(self.codes), _p(self.mags))

    @classmethod
    def init(cls, metric, st, dim, codes, mags, root_row, num_levels=9, neighbors_count=32, level0_neighbors_count=64):
        """the root on every level; level 0 holds unlinked nodes for rows 0..root_row"""
        h = lib().ig_init(int(metric), int(st), dim, root_row, root_row + 1, num_levels, neighbors_count, level0_neighbors_count)
        return cls(h, metric, st, dim, num_levels, neighbors_count, level0_neighbors_count, root_row, codes, mags)

    @classmethod
    def from_graph(cls, metric, st, dim, codes, mags, g):
        """a graph as cdb_index_set_graph takes it (dict of read_graph), slot state derived as on a load from storage"""
        L1 = g["num_levels"] + 1
        keep = [np.ascontiguousarray(a, dtype=np.uint32) for k in ("node_row", "adj", "child") for a in g[k]]
        nr, ad, ch = keep[:L1], keep[L1:2 * L1], keep[2 * L1:]
        cnt = np.array([a.size for a in nr], dtype=np.uint32)
        tbl = [(C.c_void_p * L1)(*[a.ctypes.data for a in t]) for t in (nr, ad, ch)]
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        mags = np.ascontiguousarray(mags, dtype=np.float32)
        h = lib().ig_from_graph(int(metric), int(st), dim, _p(codes), _p(mags), g["root_row"], g["entry"], g["num_levels"],
                                g["neighbors_count"], g["level0_neighbors_count"], _p(cnt), *[C.cast(t, C.c_void_p) for t in tbl])
        return cls(h, metric, st, dim, g["num_levels"], g["neighbors_count"], g["level0_neighbors_count"], g["root_row"], codes, mags)

    def insert(self, first, count, ef_construction=128, shortlist_size=64, seed=1, max_level=None):
        """index_embeddings for rows [first, first+count) of the current table -> failed u8[count]"""
        failed = np.zeros(max(count, 1), dtype=np.uint8)
        lv = None if max_level is None else np.ascontiguousarray(max_level, dtype=np.uint8)
        lib().ig_insert_rows(self.h, first, count, None if lv is None else _p(lv), seed, ef_construction, shortlist_size, _p(failed))
        return failed[:count]

    def export(self):
        """-> dict like DenseIndex.read_graph() plus simkey / lowest_idx / lowest_key per level"""
        L = lib()
        out = dict(num_levels=self.num_levels, neighbors_count=self.nbrs, level0_neighbors_count=self.nbrs0, entry=int(L.ig_entry(self.h)),
                   root_row=self.root_row, node_row=[], adj=[], child=[], simkey=[], lowest_idx=[], lowest_key=[])
        for lv in range(self.num_levels + 1):
            c = int(L.ig_level_count(self.h, lv))
            nb = self.nbrs0 if lv == 0 else self.nbrs
            a = [np.zeros(c, np.uint32), np.zeros(c * nb, np.uint32), np.zeros(c, np.uint32), np.zeros(c * nb, np.uint32),
                 np.zeros(c, np.uint32), np.zeros(c, np.uint32)]
            L.ig_level_export(self.h, lv, *[_p(x) for x in a])
            for key, x in zip(("node_row", "adj", "child", "simkey", "lowest_idx", "lowest_key"), a):
                out[key].append(x)
        return out

    def search_batch(self, raw, queries, k, lo=-1.0, hi=1.0, ef_search=256, shortlist_size=64):
        """search_internal -> (ids, scores, counts, err, evals, pops); raw = f32 rows of the whole table (root row included)"""
        raw = np.ascontiguousarray(raw, dtype=np.float32)
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        nq = queries.shape[0]
        ids = np.zeros((nq, k), np.uint32)
        scores = np.zeros((nq, k), np.float32)
        counts = np.zeros(nq, np.uint32)
        err = np.zeros(nq, np.uint8)
        ev, pp = C.c_uint64(0), C.c_uint64(0)
        lib().ig_search_batch(self.h, _p(raw), _p(queries), nq, lo, hi, ef_search, shortlist_size, k, _p(ids), _p(scores),
                              _p(counts), _p(err), C.byref(ev), C.byref(pp))
        return ids, scores, counts, err, ev.value, pp.value

    def close(self):
        if self.h:
            lib().ig_free(self.h)
            self.h = None

    __del__ = close


def slot_scores(metric, simkey, adj):
    """order keys -> the f32 similarity the library reports per slot (0 for empty slots)"""
    k = np.asarray(simkey, dtype=np.uint32)
    if int(metric) in (po.METRIC_EUCLIDEAN, po.METRIC_HAMMING):
        k = ~k
    bits = np.where(k & 0x80000000, k & 0x7FFFFFFF, ~k).astype(np.uint32)
    bits[np.asarray(adj) == 0xFFFFFFFF] = 0
    return bits.view(np.float32)


def reload_lowest(keys, adj, nb, min_key, max_key):
    """ProbNode::new_with_neighbors_and_versions (prob_node.rs:155-169) restated per node: the first empty slot gives
    (slot, MetricResult::min), else the first slot with a strictly lower similarity, scanning from MetricResult::max"""
    keys, adj = np.asarray(keys).reshape(-1, nb), np.asarray(adj).reshape(-1, nb)
    li, lk = np.zeros(len(adj), np.uint32), np.zeros(len(adj), np.uint32)
    for i in range(len(adj)):
        idx, key = 0, max_key
        for s in range(nb):
            if adj[i, s] == 0xFFFFFFFF:
                idx, key = s, min_key
                break
            if keys[i, s] < key:
                idx, key = s, int(keys[i, s])
        li[i], lk[i] = idx, key
    return li, lk


def min_max_keys(metric):
    L = po.lib()
    if int(metric) == po.METRIC_COSINE:
        return int(L.orc_order_key(int(metric), -1.0)), int(L.orc_order_key(int(metric), 2.0))
    return int(L.orc_order_key(int(metric), float("-inf"))), int(L.orc_order_key(int(metric), float("inf")))
