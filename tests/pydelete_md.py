"""ctypes binding of tests/hnsw_delete_md_oracle.c (TEST INFRASTRUCTURE ONLY): the replica oracle's builder state with
inserts continued and delete_embedding restated for graphs with metadata (cdb_index_delete_rows_replicas).  The shared
object is compiled on first use into a temporary directory (keyed by the sources' contents) and links the checker library
oracle/libcosdata_oracle.so."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po
from oracle import pyhnsw, pymeta

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "hnsw_delete_md_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    po.lib()   # builds oracle/libcosdata_oracle.so if needed
    h = hashlib.sha256()
    for p in [_SRC] + [os.path.join(_ORACLE, f) for f in ("metadata_oracle.c", "metadata_oracle.h", "hnsw_build_internal.h",
                                                          "hnsw_oracle.h", "cosdata_oracle.h")]:
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), f"cdb_delete_md_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-mpopcnt", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-fPIC", "-shared", "-std=gnu11", "-Wl,-Bsymbolic", "-I", _ORACLE, "-I", _HERE, "-o", tmp, _SRC, "-L", _ORACLE,
                        "-lcosdata_oracle", f"-Wl,-rpath,{_ORACLE}", "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, u32 = C.c_void_p, C.c_uint32
    L.mdo_new.restype = vp
    L.mdo_new.argtypes = [C.c_int, C.c_int, C.c_size_t, vp, vp, C.c_size_t, vp, vp, u32, u32, u32, u32, u32, u32, u32]
    L.mdo_free.restype = None
    L.mdo_free.argtypes = [vp]
    L.mdo_insert.restype = None
    L.mdo_insert.argtypes = [vp, C.POINTER(pymeta._ReplicaList), u32, u32, vp]
    L.mdo_delete_rows.restype = None
    L.mdo_delete_rows.argtypes = [vp, vp, u32, u32, vp, vp]
    L.mdo_count.restype = u32
    L.mdo_count.argtypes = [vp, u32]
    L.mdo_export.restype = None
    L.mdo_export.argtypes = [vp, u32] + [vp] * 9
    L.mdo_slot_calc.restype = None
    L.mdo_slot_calc.argtypes = [C.POINTER(pymeta._MdGraph), u32, vp, vp]
    L.mdo_order_keys.restype = None
    L.mdo_order_keys.argtypes = [C.c_int, vp, vp, C.c_size_t]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def order_keys(metric, scores):
    s = np.ascontiguousarray(scores, dtype=np.float32)
    out = np.zeros(s.size, np.uint32)
    lib().mdo_order_keys(int(metric), _p(s), _p(out), s.size)
    return out


def slot_calc(mg, level):
    """calculate(x, y) of every filled slot of `level` of a pymeta.MdGraph (x the Metadata end of a Pseudo-Metadata edge)
    -> (scores f32[cnt*nb], rc i32[cnt*nb], -1 on empty slots)"""
    g = mg.cstruct()
    size = mg.fg.adj[level].size
    out, rc = np.zeros(size, np.float32), np.zeros(size, np.int32)
    lib().mdo_slot_calc(C.byref(g), level, _p(out), _p(rc))
    return out, rc


class Graph:
    """the replica oracle's builder state: roots, then inserts and deletes in call order.  codes / mags cover every vector row
    the calls will name and md_bits / md_mags every Metadata row (rows appended later are simply not named before)."""

    def __init__(self, metric, st, dim, codes, mags, md_bits, md_mags, num_levels, nbrs, nbrs0, main_root_row, main_root_md,
                 pseudo_root_row, pseudo_root_md):
        self.metric, self.st, self.dim = int(metric), int(st), dim
        self.codes = np.ascontiguousarray(codes, dtype=np.uint8)
        self.mags = np.ascontiguousarray(mags, dtype=np.float32)
        self.md_bits = np.ascontiguousarray(md_bits, dtype=np.int32)
        self.md_mags = np.ascontiguousarray(md_mags, dtype=np.float32)
        self.num_levels, self.nbrs, self.nbrs0 = num_levels, nbrs, nbrs0
        self.main_root_row, self.pseudo_root_row = int(main_root_row), int(pseudo_root_row)
        self.deleted = np.zeros(self.mags.size, np.uint8)
        self.h = lib().mdo_new(self.metric, self.st, dim, _p(self.codes), _p(self.mags), self.md_bits.shape[1], _p(self.md_bits),
                               _p(self.md_mags), num_levels, nbrs, nbrs0, int(main_root_row), int(main_root_md) & 0xFFFFFFFF,
                               int(pseudo_root_row), int(pseudo_root_md))

    def insert(self, row, node_id, base_id, md_row, max_level, ef_construction, shortlist_size=64):
        """more list entries (row 0xFFFFFFFF = the pseudo root's vector) -> failed u8[n]"""
        row = np.where(np.asarray(row) == 0xFFFFFFFF, self.pseudo_root_row, row).astype(np.uint32)
        rl = pymeta.ReplicaList(row, node_id, base_id, md_row, max_level, self.main_root_row, 0, self.pseudo_root_row, 0)
        failed = np.zeros(max(row.size, 1), np.uint8)
        lib().mdo_insert(self.h, C.byref(rl.cstruct()), ef_construction, shortlist_size, _p(failed))
        return failed[: row.size]

    def delete(self, rows, shortlist_size=64):
        """delete_embedding for vector rows, one at a time in list order -> status u8[len(rows)]"""
        r = np.ascontiguousarray(rows, dtype=np.uint32)
        st = np.zeros(max(r.size, 1), np.uint8)
        lib().mdo_delete_rows(self.h, _p(r), r.size, shortlist_size, _p(self.deleted), _p(st))
        return st[: r.size]

    def export(self):
        """dict of per-level arrays: node_row, child, node_id, node_md, lowest_idx, lowest_key, ins, adj, simkey"""
        keys = ("node_row", "child", "node_id", "node_md", "lowest_idx", "lowest_key", "ins", "adj", "simkey")
        e = {k: [] for k in keys}
        for lv in range(self.num_levels + 1):
            cnt = lib().mdo_count(self.h, lv)
            nb = self.nbrs0 if lv == 0 else self.nbrs
            arrs = [np.zeros(cnt * (nb if k in ("adj", "simkey") else 1), np.uint32) for k in keys]
            lib().mdo_export(self.h, lv, *[_p(a) for a in arrs])
            for k, a in zip(keys, arrs):
                e[k].append(a)
        return e

    def md_graph(self):
        """the current graph as a pymeta.MdGraph (for the search oracle)"""
        e = self.export()
        fg = pyhnsw.FlatGraph(self.metric, self.st, self.dim, self.codes, self.mags, self.main_root_row, self.num_levels, self.nbrs,
                              self.nbrs0, 0, e["node_row"], e["adj"], e["child"])
        return pymeta.MdGraph(fg, self.md_bits, self.md_mags, e["node_id"], e["node_md"], 1)

    def close(self):
        if self.h:
            lib().mdo_free(self.h)
            self.h = None

    def __del__(self):
        self.close()
