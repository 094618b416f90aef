"""ctypes binding of tests/tfidf_oracle.c (TEST INFRASTRUCTURE ONLY): the CPU restatement of the reference's TF-IDF / BM25
index -- VersionedVec lists with version segments, N, get_idf with log1pf, search_bm25's 512 buckets and total_cmp sort, in
two summation orders (`query`, the GPU contract, and `heap`, the reference's BinaryHeap).  Compiled on first use into a
temporary directory (keyed by the source's contents) with -ffp-contract=off -fno-fast-math, like tests/pysparse.py."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "tfidf_oracle.c")
_lib = None
MODES = {"query": 0, "heap": 1}


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as f:
        h = hashlib.sha256(f.read()).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), f"cdb_tfidf_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared", "-std=gnu11",
                        "-o", tmp, _SRC, "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.to_create.restype = vp
    L.to_create.argtypes = [u32]
    L.to_destroy.argtypes = [vp]
    L.to_append.argtypes = [vp, vp, vp, vp, vp, u64, u32]
    L.to_delete.argtypes = [vp, vp, u64, u32]
    L.to_term_stats.restype = u32
    L.to_term_stats.argtypes = [vp, vp, u64, vp, vp]
    L.to_scores.restype = C.c_int
    L.to_scores.argtypes = [vp, C.c_int, vp, u64, vp, vp, vp, vp]
    L.to_search.argtypes = [vp, C.c_int, vp, vp, u32, u32, vp, vp, vp, vp]
    L.to_idf.restype = C.c_float
    L.to_idf.argtypes = [u32, u32]
    L.to_rows.restype = u64
    L.to_rows.argtypes = [vp]
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def idf(n_docs, df):
    return np.float32(lib().to_idf(n_docs, df))


class Oracle:
    """the reference's index state, fed the same append / delete calls as cdb_tfidf_index"""

    def __init__(self, id_base=0):
        self.h = lib().to_create(id_base)

    def close(self):
        if self.h:
            lib().to_destroy(self.h)
            self.h = None

    __del__ = close

    def append(self, csr, version=0, counted=None):
        o, h, v = [np.ascontiguousarray(a, dtype=t) for a, t in zip(csr, (np.uint64, np.uint32, np.float32))]
        c = None if counted is None else np.ascontiguousarray(counted, dtype=np.uint8)
        lib().to_append(self.h, _p(o), _p(h), _p(v), _p(c), len(o) - 1, version)

    def delete(self, rows, version=0):
        r = np.ascontiguousarray(np.atleast_1d(rows), dtype=np.uint32)
        lib().to_delete(self.h, _p(r), r.size, version)

    def term_stats(self, hashes):
        hs = np.ascontiguousarray(np.atleast_1d(hashes), dtype=np.uint32)
        df = np.zeros(max(hs.size, 1), np.uint32)
        f = np.zeros(max(hs.size, 1), np.float32)
        n = lib().to_term_stats(self.h, _p(hs), hs.size, _p(df), _p(f))
        return df[:hs.size], f[:hs.size], n

    def scores(self, query, mode="query"):
        """one query over every row -> (score f32[n], touched bool[n], matches u32[n], sum of |products| f64[n], panic)"""
        q = np.ascontiguousarray(query, dtype=np.uint32)
        n = int(lib().to_rows(self.h))
        acc = np.zeros(max(n, 1), np.float32)
        t = np.zeros(max(n, 1), np.uint8)
        m = np.zeros(max(n, 1), np.uint32)
        s = np.zeros(max(n, 1), np.float64)
        panic = lib().to_scores(self.h, MODES[mode], _p(q), q.size, _p(acc), _p(t), _p(m), _p(s))
        return acc[:n], t[:n].astype(bool), m[:n], s[:n], bool(panic)

    def search(self, queries, k=0, mode="query"):
        """queries: (offsets, hashes) -> ids u32[nq][kout], scores f32[nq][kout], counts u32[nq], panic bool[nq]"""
        qo, qh = np.ascontiguousarray(queries[0], dtype=np.uint64), np.ascontiguousarray(queries[1], dtype=np.uint32)
        nq = len(qo) - 1
        kout = 512 if k == 0 or k > 512 else k
        ids = np.zeros((max(nq, 1), kout), np.uint32)
        scores = np.zeros((max(nq, 1), kout), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        panic = np.zeros(max(nq, 1), np.uint8)
        lib().to_search(self.h, MODES[mode], _p(qo), _p(qh), nq, k, _p(ids), _p(scores), _p(counts), _p(panic))
        return ids[:nq], scores[:nq], counts[:nq], panic[:nq].astype(bool)
