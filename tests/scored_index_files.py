"""Test helpers for graphs loaded from the reference's index files with their stored slot similarities.

write_scored_index_dir restates the reference's serializers (as tests/test_index_files.py does) for a finished index, but
writes into every neighbour entry the MetricResult that add_neighbor kept for the slot -- tag by metric and the real
similarity -- instead of a placeholder, so that cdb_index_set_graph_slot_scores can attach them.

LoadedOracle binds tests/hnsw_loaded_md_oracle.c: the replica oracle's builder state reloaded from level arrays and stored
slot values, on which the insert and delete oracles continue."""
import ctypes as C
import hashlib
import os
import struct
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po
from oracle import pyhnsw, pymeta
from tests import pydelete_md
from tests.test_prop_file import enc_metadata_record, enc_record

NONE32 = 0xFFFFFFFF
METRIC_TAG = {0: 0, 1: 2, 2: 3, 3: 4}   # CDB_METRIC_* -> MetricResult tag (CosineSimilarity, Euclidean, Hamming, DotProduct)


def write_scored_index_dir(directory, st, dim, codes, mags, g, node_id, node_md, md_bits, md_mags, scores, tag, pseudo_entry=None,
                           row_ids=None, seed=0):
    """g: read_graph()-style dict (num_levels, neighbors_count, level0_neighbors_count, entry, node_row, adj, child);
    scores[L]: the similarity of every slot (empty slots ignored); tag: the MetricResult tag written with every filled slot.
    pseudo_entry None: a collection without a metadata schema (no Metadata records, no pseudo link).  row_ids: the prop id of
    each Storage record (default: the id of the row's base node).  Storage records are written in row order, so a node's
    row is its record ordinal.  -> (root_link, pseudo_link)"""
    os.makedirs(directory, exist_ok=True)
    rng = np.random.default_rng(seed)
    L1 = g["num_levels"] + 1
    nbs = [g["level0_neighbors_count"]] + [g["neighbors_count"]] * g["num_levels"]
    with_md = pseudo_entry is not None
    value_loc, md_loc = {}, {}
    if row_ids is None:
        row_ids = {}
        for lv in range(L1):
            for i in range(g["node_row"][lv].size):
                row, md = int(g["node_row"][lv][i]), int(node_md[lv][i])
                if md == NONE32 or md_mags[md] == 0.0 or row not in row_ids:
                    row_ids.setdefault(row, int(node_id[lv][i]))
    with open(os.path.join(directory, "prop.data"), "wb") as f:
        for row in range(codes.shape[0]):
            rec = enc_record(int(row_ids.get(row, 4_000_000 + row)) if isinstance(row_ids, dict) else int(row_ids[row]), st,
                             mags[row], codes[row], dim)
            value_loc[row] = (f.tell(), len(rec))
            f.write(rec)
            if with_md:
                for lv in range(L1):
                    for i in np.flatnonzero(g["node_row"][lv] == row):
                        nid, md = int(node_id[lv][i]), int(node_md[lv][i])
                        if md != NONE32 and nid not in md_loc:
                            rec = enc_metadata_record(nid, md_mags[md], md_bits[md])
                            md_loc[nid] = (f.tell(), len(rec))
                            f.write(rec)
    nodes = [(lv, i) for lv in range(L1) for i in range(g["node_row"][lv].size)]
    link = {n: int(s) * 8 for n, s in zip(nodes, rng.permutation(len(nodes)))}
    parent = {}
    for lv in range(1, L1):
        for j in range(g["node_row"][lv].size):
            parent[(lv - 1, int(g["child"][lv][j]))] = (lv, j)
    files = {0: bytearray(), 1: bytearray()}
    place = {}
    for n in nodes:
        size = 31 + 13 * nbs[n[0]]
        fid = int(rng.integers(0, 2))
        place[n] = (fid, len(files[fid]))
        files[fid] += bytes(size)
    for n in nodes:
        lv, i = n
        nb = nbs[lv]
        row, nid, md = int(g["node_row"][lv][i]), int(node_id[lv][i]), int(node_md[lv][i])
        buf = struct.pack("<BI", lv, 7) + struct.pack("<II", *value_loc[row])
        buf += struct.pack("<II", *md_loc[nid]) if (with_md and md != NONE32) else b"\xff" * 8
        buf += struct.pack("<I", link[parent[n]] if n in parent else NONE32)
        buf += struct.pack("<I", link[(lv - 1, int(g["child"][lv][i]))] if lv > 0 else NONE32)
        buf += struct.pack("<H", nb)
        for s in range(nb):
            t = int(g["adj"][lv][i * nb + s])
            if t == NONE32:
                buf += b"\xff" * 13
            else:
                buf += struct.pack("<IIB", int(node_id[lv][t]), link[(lv, t)], tag) + np.float32(scores[lv][i * nb + s]).tobytes()
        fid, off = place[n]
        files[fid][off:off + len(buf)] = buf
    ptr = bytearray(8 * len(nodes))
    for n in nodes:
        fid, off = place[n]
        ptr[link[n]:link[n] + 8] = struct.pack("<II", off, fid)
    open(os.path.join(directory, "nodes.ptr"), "wb").write(bytes(ptr))
    for fid, b in files.items():
        open(os.path.join(directory, f"{fid}.index"), "wb").write(bytes(b))
    top = g["num_levels"]
    return link[(top, g["entry"])], (NONE32 if pseudo_entry is None else link[(top, pseudo_entry)])


_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hnsw_loaded_md_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    po.lib()
    here = os.path.dirname(_SRC)
    orc_dir = os.path.join(os.path.dirname(here), "oracle")
    h = hashlib.sha256()
    for p in [_SRC, pydelete_md._SRC] + [os.path.join(orc_dir, f) for f in ("metadata_oracle.c", "metadata_oracle.h",
                                                                           "hnsw_build_internal.h", "hnsw_oracle.h", "cosdata_oracle.h")]:
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), f"cdb_loaded_md_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-mpopcnt", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-fPIC", "-shared", "-std=gnu11", "-Wl,-Bsymbolic", "-I", orc_dir, "-I", here, "-o", tmp, _SRC, "-L", orc_dir,
                        "-lcosdata_oracle", f"-Wl,-rpath,{orc_dir}", "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, u32 = C.c_void_p, C.c_uint32
    L.mdo_load.restype = vp
    L.mdo_load.argtypes = [C.c_int, C.c_int, C.c_size_t, vp, vp, C.c_size_t, vp, vp, u32, u32, u32] + [vp] * 8
    L.mdo_lowest.restype = None
    L.mdo_lowest.argtypes = [vp, vp, u32, u32, u32, C.POINTER(u32), C.POINTER(u32)]
    L.mdo_key_range.restype = None
    L.mdo_key_range.argtypes = [C.c_int, C.POINTER(u32), C.POINTER(u32)]
    for name in ("mdo_free", "mdo_insert", "mdo_delete_rows", "mdo_count", "mdo_export", "mdo_order_keys"):
        f, src = getattr(L, name), getattr(pydelete_md.lib(), name)
        f.restype, f.argtypes = src.restype, src.argtypes
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _table(arrs, dtype):
    keep = [np.ascontiguousarray(a, dtype=dtype) for a in arrs]
    return keep, (C.c_void_p * len(keep))(*[a.ctypes.data for a in keep])


def lowest(adj, simkey, metric):
    """mdo_lowest for one node -> (lowest_idx, lowest_key)"""
    a, k = np.ascontiguousarray(adj, np.uint32), np.ascontiguousarray(simkey, np.uint32)
    lo, hi = C.c_uint32(), C.c_uint32()
    lib().mdo_key_range(int(metric), C.byref(lo), C.byref(hi))
    li, lk = C.c_uint32(), C.c_uint32()
    lib().mdo_lowest(_p(a), _p(k), a.size, lo.value, hi.value, C.byref(li), C.byref(lk))
    return li.value, lk.value


def key_range(metric):
    lo, hi = C.c_uint32(), C.c_uint32()
    lib().mdo_key_range(int(metric), C.byref(lo), C.byref(hi))
    return lo.value, hi.value


class LoadedOracle(pydelete_md.Graph):
    """pydelete_md.Graph whose state is reloaded from level arrays and stored slot values (mdo_load).  The arrays are in the
    numbering the GPU holds them (entry / pseudo_entry: top-level indices; pseudo_entry None: no pseudo root).  They are
    renumbered into the oracle's layout -- main root, pseudo root (or an isolated placeholder), then every other node in the
    order it had -- keeping each loaded node's list position (its level-0 index); export() maps back to the GPU numbering."""

    def __init__(self, metric, st, dim, codes, mags, md_bits, md_mags, num_levels, nbrs, nbrs0, node_row, node_id, node_md, adj, child,
                 scores, entry=0, pseudo_entry=1):
        self.metric, self.st, self.dim = int(metric), int(st), dim
        self.codes = np.ascontiguousarray(codes, dtype=np.uint8)
        self.mags = np.ascontiguousarray(mags, dtype=np.float32)
        self.md_bits = np.ascontiguousarray(md_bits, dtype=np.int32)
        self.md_mags = np.ascontiguousarray(md_mags, dtype=np.float32)
        self.num_levels, self.nbrs, self.nbrs0 = num_levels, nbrs, nbrs0
        self.has_pseudo = pseudo_entry is not None
        L1, top = num_levels + 1, num_levels
        nbs = [nbrs0] + [nbrs] * num_levels
        # the roots' local indices, down the child links
        r0, r1 = [0] * L1, [None] * L1
        r0[top], r1[top] = int(entry), (int(pseudo_entry) if self.has_pseudo else None)
        for lv in range(top, 0, -1):
            r0[lv - 1] = int(child[lv][r0[lv]])
            r1[lv - 1] = int(child[lv][r1[lv]]) if self.has_pseudo else None
        self.main_root_row = int(node_row[top][r0[top]])
        self.pseudo_root_row = int(node_row[top][r1[top]]) if self.has_pseudo else None
        self.deleted = np.zeros(self.mags.size, np.uint8)
        self.to_gpu, self.loaded_cnt = [], []     # per level: oracle index -> GPU index (-1: the placeholder)
        arrs = {k: [] for k in ("node_row", "node_id", "node_md", "adj", "child", "scores")}
        for lv in range(L1):
            cnt, nb = node_row[lv].size, nbs[lv]
            rest = [i for i in range(cnt) if i != r0[lv] and i != r1[lv]]
            order = np.array([r0[lv], r1[lv] if self.has_pseudo else -1] + rest, np.int64)
            inv = np.zeros(cnt + 1, np.int64)
            inv[order[order >= 0]] = np.flatnonzero(order >= 0)
            inv[cnt] = NONE32
            src = np.where(order >= 0, order, r0[lv])                     # the placeholder copies the main root's row
            a = adj[lv].reshape(cnt, nb)[src].astype(np.int64)
            a = np.where(a == NONE32, cnt, a)
            a = inv[a].astype(np.uint32)
            sc = np.asarray(scores[lv], np.float32).reshape(cnt, nb)[src].copy()
            nid, nmd = node_id[lv][src].copy(), node_md[lv][src].copy()
            if not self.has_pseudo:
                a[1] = NONE32
                sc[1] = 0
                nid[1], nmd[1] = 0xFFFFFFFF - 257, NONE32
            if lv:
                ch = self._inv_below[child[lv][src].astype(np.int64)].astype(np.uint32)
                if not self.has_pseudo:
                    ch[1] = 1
            else:
                ch = np.zeros(cnt + (0 if self.has_pseudo else 1), np.uint32)
                self.pos0 = np.where(order >= 0, order, NONE32).astype(np.uint32)   # a loaded node's list position
            self._inv_below = inv
            for k, v in (("node_row", node_row[lv][src]), ("node_id", nid), ("node_md", nmd), ("adj", a.ravel()), ("child", ch),
                         ("scores", sc.ravel())):
                arrs[k].append(v)
            self.to_gpu.append(order)
            self.loaded_cnt.append(order.size)
        counts = np.array([a.size for a in arrs["node_row"]], np.uint32)
        self._keep = [counts, self.pos0]
        tables = []
        for k, dt in (("node_row", np.uint32), ("node_id", np.uint32), ("node_md", np.uint32), ("adj", np.uint32), ("child", np.uint32),
                      ("scores", np.float32)):
            keep, t = _table(arrs[k], dt)
            self._keep.append(keep)
            tables.append(t)
        self.h = lib().mdo_load(self.metric, self.st, dim, _p(self.codes), _p(self.mags), self.md_bits.shape[1], _p(self.md_bits),
                                _p(self.md_mags), num_levels, nbrs, nbrs0, _p(counts), *[C.cast(t, C.c_void_p) for t in tables],
                                _p(self.pos0))
        if not self.h:
            raise ValueError("mdo_load refused the layout")

    def insert(self, row, node_id, base_id, md_row, max_level, ef_construction, shortlist_size=64):
        row = np.asarray(row)
        if not self.has_pseudo:   # as cdb_index_insert_graph_replicas on a graph without a pseudo root
            md = np.asarray(md_row)
            if (row == NONE32).any() or (self.md_mags[md[md != NONE32]] != 0).any():
                raise ValueError("no pseudo root: pseudo replicas and Metadata with mag != 0 are refused")
        row = np.where(row == NONE32, self.pseudo_root_row if self.has_pseudo else 0, row).astype(np.uint32)
        rl = pymeta.ReplicaList(row, node_id, base_id, md_row, max_level, self.main_root_row, 0,
                                self.pseudo_root_row if self.has_pseudo else self.main_root_row, 0)
        failed = np.zeros(max(row.size, 1), np.uint8)
        lib().mdo_insert(self.h, C.byref(rl.cstruct()), ef_construction, shortlist_size, _p(failed))
        return failed[: row.size]

    def delete(self, rows, shortlist_size=64):
        r = np.ascontiguousarray(rows, dtype=np.uint32)
        st = np.zeros(max(r.size, 1), np.uint8)
        lib().mdo_delete_rows(self.h, _p(r), r.size, shortlist_size, _p(self.deleted), _p(st))
        return st[: r.size]

    def export(self):
        """per-level arrays in the GPU's numbering (nodes inserted after the load follow the loaded ones in both):
        node_row, child, node_id, node_md, lowest_idx, lowest_key, ins, adj, simkey"""
        keys = ("node_row", "child", "node_id", "node_md", "lowest_idx", "lowest_key", "ins", "adj", "simkey")
        e = {k: [] for k in keys}
        below = None
        for lv in range(self.num_levels + 1):
            cnt = lib().mdo_count(self.h, lv)
            nb = self.nbrs0 if lv == 0 else self.nbrs
            arrs = [np.zeros(cnt * (nb if k in ("adj", "simkey") else 1), np.uint32) for k in keys]
            lib().mdo_export(self.h, lv, *[_p(a) for a in arrs])
            loaded = self.to_gpu[lv]
            shift = 0 if self.has_pseudo else 1
            gpu_of = np.concatenate([loaded, np.arange(loaded.size, cnt) - shift]).astype(np.int64)   # oracle -> GPU index
            keep = gpu_of >= 0
            n_gpu = int(keep.sum())
            perm = np.zeros(n_gpu, np.int64)
            perm[gpu_of[keep]] = np.flatnonzero(keep)                       # GPU index -> oracle index
            remap = np.concatenate([np.where(keep, gpu_of, -1), [NONE32]])
            for k, a in zip(keys, arrs):
                if k in ("adj", "simkey"):
                    a = a.reshape(cnt, nb)[perm]
                    if k == "adj":
                        a = remap[np.where(a == NONE32, cnt, a).astype(np.int64)]
                        assert (a >= 0).all()                                # nothing links the placeholder
                    a = a.astype(np.uint32).ravel()
                else:
                    a = a[perm]
                    if k == "child" and lv:
                        a = below[a.astype(np.int64)].astype(np.uint32)
                e[k].append(a)
            below = remap
        return e

    def close(self):
        if self.h:
            lib().mdo_free(self.h)
            self.h = None
