"""Hybrid search over mixed batches: one cdb_hybrid_search_batch_mixed[_sharded] call against the split-by-kind composition
a shim needs without it (one two-source host call per kind present, cdb_hybrid_search_batch[_sharded], and the rows put
back in request order), at batch 1 / 64 / 1024 and top_k = 10.
  mixed_ms   the mixed host call, wall clock around the synchronising call
  split_ms   the two-source host calls plus the reassembly, wall clock
Batches: kinds in equal thirds, shuffled ("thirds"), and for contrast one kind, dense + sparse ("one_kind").  Targets:
the single index, a `--shards`-slot group (one card per slot when there are that many cards, else loopback slots on device
0) and the one-slot group over the whole corpus.  Corpora, all seeded, as tools/bench_hybrid.py and
tools/bench_hybrid_sharded.py: 1M x 768 f16 dense rows (synthetic stream, raw f32 kept) with GPU-built HNSW graphs
(ef_search 128), the 1M-row sparse and TF-IDF corpora; the single index is the one-slot group's indexes.  Each timing is
the median of `--steps` calls after `--warmup`; the two forms alternate over `--repeats` runs and each JSON line reports
the min and max of the run medians.  The last timed rows of both forms are compared bit for bit on every query.  Prints
the card and its power limit, then one JSON line per (target, batch kind, batch).

    python tools/bench_hybrid_mixed.py [--rows 1000000] [--shards 2] [--steps 10] [--warmup 2] [--repeats 3]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cosdata_b200 as cdb  # noqa: E402
from cosdata_b200 import _lib  # noqa: E402
from cosdata_b200.api import _query_csr, sparse_csr  # noqa: E402
from cosdata_b200.sharding import shard_range  # noqa: E402
from bench_hybrid_sharded import CHUNK, DENSE, build_group, card  # noqa: E402
from tests.pyhybrid_mixed import KIND_SOURCES  # noqa: E402
from tests.sparse_data import concat_csr, zipf_csr  # noqa: E402
from tests.tfidf_data import zipf_docs, zipf_queries  # noqa: E402

DIM = 768
TOP_K = 10
SP_OPTS = cdb.SparseSearchOptions(0, 0.0)


def csr_rows(c):
    o, d, v = c
    return [list(zip(d[int(o[i]):int(o[i + 1])].tolist(), v[int(o[i]):int(o[i + 1])].tolist())) for i in range(len(o) - 1)]


class Request:
    """one batch's host arrays for the mixed call and for each kind's two-source call, built once so that the timings hold
    the library calls and the reassembly only"""

    def __init__(self, kinds, dq, sq, tq, handles=None, dense_params=None):
        self.kinds, self.b = kinds, kinds.size
        self.keep = [kinds]
        group = handles is None
        w = 6 * TOP_K
        self.out = [np.zeros((self.b, w), np.uint32), np.zeros((self.b, w), np.float32), np.zeros(self.b, np.uint32), np.zeros(self.b, np.uint8)]
        _, batches = cdb.split_mixed(kinds, dq, sq, tq)
        m = _lib.HybridGroupMixedSources() if group else _lib.HybridMixedSources()
        m.kinds = kinds.ctypes.data
        m.dense_params, m.sparse_params = dense_params, SP_OPTS.params()
        if group:
            m.dense_id_stride = 1
        else:
            m.dense, m.sparse, m.tfidf = handles
        self._fill(m, batches, mixed=True)
        self.mixed = m
        self.parts = []   # (rows, sources struct, outputs)
        for kind in np.unique(kinds).tolist():
            rows = np.flatnonzero(kinds == kind)
            names = KIND_SOURCES[kind]
            s = _lib.HybridGroupSources() if group else _lib.HybridSources()
            s.dense_params, s.sparse_params = dense_params, SP_OPTS.params()
            sub = {"dense": dq[rows], "sparse": [sq[i] for i in rows], "tfidf": [tq[i] for i in rows]}
            if group:
                s.use_dense, s.use_sparse, s.use_tfidf = ("dense" in names), ("sparse" in names), ("tfidf" in names)
                s.dense_id_stride = 1
            else:
                s.dense, s.sparse, s.tfidf = (h if n in names else None for h, n in zip(handles, ("dense", "sparse", "tfidf")))
            self._fill(s, {n: sub[n] for n in names}, mixed=False)
            out = [np.zeros((rows.size, w), np.uint32), np.zeros((rows.size, w), np.float32), np.zeros(rows.size, np.uint32),
                   np.zeros(rows.size, np.uint8)]
            self.parts.append((rows, s, out))

    def _fill(self, s, batches, mixed):
        if "dense" in batches:
            q = np.ascontiguousarray(batches["dense"], dtype=np.float32)
            s.dense_queries = q.ctypes.data
            self.keep.append(q)
            if mixed:
                s.n_dense = q.shape[0]
        if "sparse" in batches:
            o, d, v = sparse_csr(batches["sparse"])
            s.sparse_offsets, s.sparse_dims, s.sparse_values = o.ctypes.data, d.ctypes.data, v.ctypes.data
            self.keep += [o, d, v]
            if mixed:
                s.n_sparse = len(o) - 1
        if "tfidf" in batches:
            o, h = _query_csr(batches["tfidf"])
            s.tfidf_offsets, s.tfidf_hashes = o.ctypes.data, h.ctypes.data
            self.keep += [o, h]
            if mixed:
                s.n_tfidf, s.n_tfidf_hashes = len(o) - 1, int(o[-1])

    @staticmethod
    def ptrs(out):
        return [x.ctypes.data for x in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    name = card()
    print(json.dumps({"card": name, "gpus": cdb.device_count()}), flush=True)
    n, w = a.rows, a.shards
    t0 = time.perf_counter()
    sp_corpus = concat_csr([zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))])
    tf_corpus = concat_csr([zipf_docs(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))])
    devs = list(range(w)) if cdb.device_count() >= w else [0] * w
    g_w, keep_w = build_group(devs, [shard_range(n, w, r)[0] for r in range(w)] + [n], sp_corpus, tf_corpus)
    g_1, keep_1 = build_group([0], [0, n], sp_corpus, tf_corpus)
    del sp_corpus, tf_corpus
    torch.cuda.synchronize()
    print(json.dumps({"setup_s": round(time.perf_counter() - t0, 1), "rows": n, "shards": w, "loopback": devs.count(0) > 1}), flush=True)
    dense, sp, tf = keep_1
    L = _lib.load()
    dq_all = cdb.synth_matrix(12, 1024, DIM)
    sq_all = csr_rows(zipf_csr(7, 1024, mean_pairs=40))
    tq_all = zipf_queries(7, 1024, vocab=1_000_000)
    targets = {"single": None, f"group{w}": g_w, "group1": g_1}

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            fn()
            ts.append(1e3 * (time.perf_counter() - t0))
        return float(np.median(ts))

    for target, g in targets.items():
        for batch_kind in ("thirds", "one_kind"):
            for b in (1, 64, 1024):
                rng = np.random.default_rng(b)
                if batch_kind == "thirds":
                    kinds = (np.arange(b) % 3).astype(np.uint8)
                    rng.shuffle(kinds)
                else:
                    kinds = np.zeros(b, np.uint8)
                handles = None if g else (dense._h, sp.h, tf.h)
                req = Request(kinds, dq_all[:b], sq_all[:b], tq_all[:b], handles, dense.params(0, **DENSE))

                def mixed():
                    o = Request.ptrs(req.out)
                    if g is None:
                        rc = L.cdb_hybrid_search_batch_mixed(C.byref(req.mixed), b, TOP_K, 60.0, *o)
                    else:
                        rc = L.cdb_hybrid_search_batch_mixed_sharded(g._h, C.byref(req.mixed), b, TOP_K, 60.0, *o)
                    assert rc == 0, L.cdb_last_error_string()

                split_out = [np.zeros_like(x) for x in req.out]

                def split():
                    for rows, s, out in req.parts:
                        o = Request.ptrs(out)
                        if g is None:
                            rc = L.cdb_hybrid_search_batch(C.byref(s), rows.size, TOP_K, 60.0, *o)
                        else:
                            rc = L.cdb_hybrid_search_batch_sharded(g._h, C.byref(s), rows.size, TOP_K, 60.0, *o)
                        assert rc == 0, L.cdb_last_error_string()
                        for full, part in zip(split_out, out):
                            full[rows] = part
                    # a dense-less kind's call leaves its error bytes alone: they are 0 from the start

                ms = {"mixed": [], "split": []}
                for _ in range(a.repeats):
                    ms["mixed"].append(timed(mixed))
                    ms["split"].append(timed(split))
                same = (np.array_equal(req.out[2], split_out[2]) and np.array_equal(req.out[0], split_out[0])
                        and np.array_equal(req.out[1].view(np.uint32), split_out[1].view(np.uint32))
                        and np.array_equal(req.out[3], split_out[3]))
                res = {"target": target, "batch_kind": batch_kind, "batch": b, "top_k": TOP_K, "card": name,
                       "mixed_ms": [round(min(ms["mixed"]), 3), round(max(ms["mixed"]), 3)],
                       "split_ms": [round(min(ms["split"]), 3), round(max(ms["split"]), 3)],
                       "split_calls": len(req.parts), "equal": bool(same)}
                print(json.dumps(res), flush=True)
                assert same, "the mixed call and the split-by-kind composition differ"
    g_w.close()
    g_1.close()
    for x in keep_w + keep_1:
        x.close()


if __name__ == "__main__":
    main()
