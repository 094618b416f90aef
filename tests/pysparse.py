"""ctypes binding of tests/sparse_oracle.c (TEST INFRASTRUCTURE ONLY): the CPU restatement of the reference's sparse inverted
index search, re-rank and sampling.  The shared object is compiled on first use into a temporary directory (keyed by the
source's contents), with the flags of oracle/Makefile that matter for parity (-ffp-contract=off -fno-fast-math).  It sits
next to the other oracles of the index writers (hnsw_insert_oracle.c, hnsw_delete_oracle.c, ...), which are built the same
way: the files under oracle/ are the frozen checker of the dense path and are not rebuilt or extended per feature."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sparse_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as f:
        h = hashlib.sha256(f.read()).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), f"cdb_sparse_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared", "-std=gnu11",
                        "-o", tmp, _SRC, "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, u32, u64, f32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float
    L.so_quantize.restype = u32
    L.so_quantize.argtypes = [f32, f32, u32]
    L.so_thresholds.argtypes = [f32, u32, C.POINTER(u32), C.POINTER(u32)]
    L.so_search.argtypes = [u32, f32, f32, C.c_int, u32, u32, u32, u64, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp]
    L.so_sample.restype = f32
    L.so_sample.argtypes = [vp, u64, f32, vp, u64, vp]
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def csr(rows):
    """list of [(dim, value), ...] -> (offsets u64, dims u32, values f32)"""
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows]) if rows else []
    dims = np.array([d for r in rows for d, _ in r], np.uint32)
    vals = np.array([v for r in rows for _, v in r], np.float32)
    return off, dims, vals


def quantize(value, ub, bits):
    return int(lib().so_quantize(float(value), float(ub), bits))


def thresholds(thr, bits):
    e, lo = C.c_uint32(0), C.c_uint32(0)
    lib().so_thresholds(float(thr), bits, C.byref(e), C.byref(lo))
    return e.value, lo.value


def search(corpus, queries, k, bits=4, ub=1.0, thr=0.0, rerank=False, factor=5, id_base=0, deleted=None):
    """corpus / queries: CSR triples (offsets, dims, values) -> ids [nq][k], scores [nq][k], counts [nq]"""
    ro, rd, rv = [np.ascontiguousarray(a) for a in corpus]
    qo, qd, qv = [np.ascontiguousarray(a) for a in queries]
    ro, qo = ro.astype(np.uint64), qo.astype(np.uint64)
    rd, qd = rd.astype(np.uint32), qd.astype(np.uint32)
    rv, qv = rv.astype(np.float32), qv.astype(np.float32)
    n, nq = len(ro) - 1, len(qo) - 1
    ids = np.zeros((nq, k), np.uint32)
    scores = np.zeros((nq, k), np.float32)
    counts = np.zeros(nq, np.uint32)
    dl = None if deleted is None else np.ascontiguousarray(deleted, dtype=np.uint8)
    lib().so_search(bits, float(ub), float(thr), 1 if rerank else 0, factor, k, id_base, n, _p(ro), _p(rd), _p(rv), _p(dl), nq,
                    _p(qo), _p(qd), _p(qv), _p(ids), _p(scores), _p(counts))
    return ids, scores, counts


def sample(values, clamp_margin_percent=1.0, prior=None, prior_values=0):
    v = np.ascontiguousarray(values, dtype=np.float32)
    counts = np.zeros(9, np.uint64)
    pr = None if prior is None else np.ascontiguousarray(prior, dtype=np.uint64)
    ub = lib().so_sample(_p(v), v.size, float(clamp_margin_percent), _p(pr), prior_values, _p(counts))
    return counts, ub
