"""Hybrid search (reciprocal-rank fusion) on one GPU, for each pairing at batch 1 / 64 / 1024 and top_k = 10:
  composed    cdb_hybrid_search_batch_device: both sub-searches overlapped on two streams, fusion on the device
  serial      the same two *_search_batch_device calls back to back on one stream, no fusion
  fuse        cdb_rrf_fuse_device alone on the two lists
  host_path   what a shim does without the fused entry point: the two host-form searches (results copied back) and a
              fusion on the host -- here tests/pyhybrid.py in Python, which is far slower than a Rust hash map would be,
              so the searches and the fusion are reported apart
Device times are CUDA events around `--steps` calls after a warm-up; host times are wall clock around calls that end in a
device synchronise.  Corpora, all seeded: 1M x 768 f16 dense rows (synthetic stream, raw f32 kept for the re-rank) with a
GPU-built HNSW graph, and the 1M-row sparse and 1M-document TF-IDF corpora of bench_sparse.py / bench_tfidf.py.  On a
32-query sample the composed results are checked against pyhybrid over the separately obtained lists.  Prints the card
and its power limit, then one JSON line per (pairing, batch).

    python tools/bench_hybrid.py [--rows 1000000] [--steps 10] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosdata_b200 as cdb  # noqa: E402
from cosdata_b200 import _lib  # noqa: E402
from tests import pyhybrid as ph  # noqa: E402
from tests.sparse_data import zipf_csr  # noqa: E402
from tests.tfidf_data import query_csr, zipf_docs, zipf_queries  # noqa: E402

CHUNK = 500_000
DIM = 768
TOP_K = 10
DENSE = {"mode": cdb.SearchMode.HNSW, "ef_search": 128, "shortlist_size": 64}
PAIRS = [("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf")]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parity-queries", type=int, default=32)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    dev = torch.device("cuda", 0)
    name = card()
    print(json.dumps({"card": name}), flush=True)
    n = a.rows
    t0 = time.perf_counter()
    dense = cdb.DenseIndex(dim=DIM, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=n + 1, keep_raw_f32=True)
    dense.append_synthetic(11, n)
    dense.build_graph(9, 32, 64, 128, 64, 4096, 7)
    sp_chunks = [zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))]
    sp = cdb.SparseIndex(quantization_bits=4, values_upper_bound=3.0, capacity_rows=n,
                         capacity_pairs=sum(len(c[1]) for c in sp_chunks))
    for c in sp_chunks:
        sp.append(c)
    del sp_chunks
    tf_chunks = [zipf_docs(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))]
    tf = cdb.TfIdfIndex(capacity_rows=n, capacity_pairs=sum(len(c[1]) for c in tf_chunks))
    for c in tf_chunks:
        tf.append(c, 1)
    del tf_chunks
    torch.cuda.synchronize()
    print(json.dumps({"setup_s": round(time.perf_counter() - t0, 1), "rows": n}), flush=True)

    dq_all = cdb.synth_matrix(12, 1024, DIM)
    sq_all = zipf_csr(7, 1024, mean_pairs=40)
    tq_all = zipf_queries(7, 1024, vocab=1_000_000)
    k3 = 3 * TOP_K
    s = torch.cuda.Stream(dev)   # a stream of its own: a NULL stream means the handle's own stream to the dense search
    L = _lib.load()

    def t(x):
        x = np.ascontiguousarray(x)
        return torch.from_numpy(x.view({np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(x.dtype, x.dtype))).to(dev)

    def dev_timed(fn):
        for _ in range(a.warmup):
            fn()
        s.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(a.steps):
            fn()
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1) / a.steps

    for pair in PAIRS:
        for b in (1, 64, 1024):
            dq = dq_all[:b]
            so = sq_all[0][:b + 1]
            sq = (so, sq_all[1][:int(so[-1])], sq_all[2][:int(so[-1])])
            tq = tq_all[:b]
            to, th = query_csr(tq)
            keep = []
            src = _lib.HybridSources()
            lists = {}          # name -> (device ids, device scores, device counts, ld, search call)

            def alloc(ld):
                x = (torch.zeros((b, ld), dtype=torch.int32, device=dev), torch.zeros((b, ld), dtype=torch.float32, device=dev),
                     torch.zeros(b, dtype=torch.int32, device=dev))
                keep.extend(x)
                return x
            if "dense" in pair:
                d_q = t(dq)
                keep.append(d_q)
                src.dense, src.dense_queries, src.dense_params = dense._h, d_q.data_ptr(), dense.params(0, **DENSE)
                ids, sc, ct = alloc(k3)
                p = dense.params(k3, **DENSE)
                lists["dense"] = (ids, ct, k3, lambda ids=ids, sc=sc, ct=ct, p=p: L.cdb_search_batch_device(
                    dense._h, d_q.data_ptr(), b, C.byref(p), ids.data_ptr(), sc.data_ptr(), ct.data_ptr(), None, C.c_void_p(s.cuda_stream)))
            if "sparse" in pair:
                d_o, d_d, d_v = t(sq[0]), t(sq[1]), t(sq[2])
                keep += [d_o, d_d, d_v]
                src.sparse, src.sparse_offsets, src.sparse_dims, src.sparse_values = sp.h, d_o.data_ptr(), d_d.data_ptr(), d_v.data_ptr()
                src.sparse_params = cdb.SparseSearchOptions(0, 0.0).params()
                ids, sc, ct = alloc(k3)
                p = cdb.SparseSearchOptions(k3, 0.0).params()
                lists["sparse"] = (ids, ct, k3, lambda ids=ids, sc=sc, ct=ct, p=p: L.cdb_sparse_search_batch_device(
                    sp.h, d_o.data_ptr(), d_d.data_ptr(), d_v.data_ptr(), b, C.byref(p), ids.data_ptr(), sc.data_ptr(), ct.data_ptr(),
                    C.c_void_p(s.cuda_stream)))
            if "tfidf" in pair:
                d_to, d_th = t(to), t(th)
                keep += [d_to, d_th]
                src.tfidf, src.tfidf_offsets, src.tfidf_hashes = tf.h, d_to.data_ptr(), d_th.data_ptr()
                ids, sc, ct = alloc(k3)
                lists["tfidf"] = (ids, ct, k3, lambda ids=ids, sc=sc, ct=ct: L.cdb_tfidf_search_batch_device(
                    tf.h, d_to.data_ptr(), d_th.data_ptr(), b, k3, ids.data_ptr(), sc.data_ptr(), ct.data_ptr(),
                    C.c_void_p(s.cuda_stream)))
            out_ids, out_sc, out_ct = alloc(6 * TOP_K)
            fa, fb = lists[pair[0]], lists[pair[1]]

            def composed():
                assert L.cdb_hybrid_search_batch_device(C.byref(src), b, TOP_K, 60.0, out_ids.data_ptr(), out_sc.data_ptr(),
                                                        out_ct.data_ptr(), None, C.c_void_p(s.cuda_stream)) == 0

            def serial():
                assert fa[3]() == 0 and fb[3]() == 0

            def fuse():
                assert L.cdb_rrf_fuse_device(0, fa[0].data_ptr(), fa[1].data_ptr(), fa[2], 1, fb[0].data_ptr(), fb[1].data_ptr(), fb[2], 1,
                                             b, 60.0, 6 * TOP_K, out_ids.data_ptr(), out_sc.data_ptr(), out_ct.data_ptr(),
                                             C.c_void_p(s.cuda_stream)) == 0
            res = {"pair": "+".join(pair), "batch": b, "top_k": TOP_K, "card": name}
            res["composed_ms"] = round(dev_timed(composed), 4)
            res["serial_ms"] = round(dev_timed(serial), 4)
            res["fuse_ms"] = round(dev_timed(fuse), 4)
            # the host path: host-form searches (queries up, results down, synchronised), then the fusion on the host
            host = {"dense": lambda: dense.batch_search(dq, k3, **DENSE)[:3],
                    "sparse": lambda: sp.batch_search(sq, cdb.SparseSearchOptions(k3, 0.0)),
                    "tfidf": lambda: tf.batch_search(tq, k3)}
            for _ in range(a.warmup):
                host[pair[0]](), host[pair[1]]()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                la, lb = host[pair[0]](), host[pair[1]]()
            res["host_searches_ms"] = round(1e3 * (time.perf_counter() - t0) / a.steps, 4)
            t0 = time.perf_counter()
            want = ph.fuse_batch(la[0], la[2], lb[0], lb[2], 60.0, ld_out=6 * TOP_K)
            res["host_python_fusion_ms"] = round(1e3 * (time.perf_counter() - t0), 4)
            # parity on a sample of the batch
            composed()
            s.synchronize()
            sel = np.arange(0, b, max(1, b // a.parity_queries))[: a.parity_queries]
            got = (out_ids.cpu().numpy().view(np.uint32), out_sc.cpu().numpy(), out_ct.cpu().numpy().view(np.uint32))
            res[f"parity_{sel.size}q"] = bool(np.array_equal(got[2][sel], want[2][sel]) and np.array_equal(got[0][sel], want[0][sel])
                                             and np.array_equal(got[1][sel].view(np.uint32), want[1][sel].view(np.uint32)))
            print(json.dumps(res), flush=True)
    dense.close()
    sp.close()
    tf.close()


if __name__ == "__main__":
    main()
