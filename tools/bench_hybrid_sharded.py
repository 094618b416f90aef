"""Hybrid search over a shard group (cdb_hybrid_search_batch_sharded[_device]) for each pairing at batch 1 / 64 / 1024 and
top_k = 10, against what a shim does without it: the two group host calls (each copies its merged list back) and the
host-form cdb_rrf_fuse (both lists copied up again, the fused list back).
  g{W}_entry_ms   host form of the group entry point, wall clock around the synchronising call
  g{W}_shim_ms    the two group host calls plus cdb_rrf_fuse, wall clock
  g1_device_ms    device form on the one-slot group, CUDA events on a side stream (no TF-IDF: the device form refuses it)
W is the group of `--shards` slots (one per card when there are that many cards, else loopback slots on device 0) and 1
the one-slot local group over the whole corpus, the route of a collection with a metadata schema on one GPU.  Corpora,
all seeded: 1M x 768 f16 dense rows (synthetic stream, raw f32 kept) with GPU-built HNSW graphs (ef_search 128), and the
1M-row sparse and TF-IDF corpora of bench_sparse.py / bench_tfidf.py, split into contiguous id ranges (dense shard r's
ids start at r * 2^21, since each graph keeps a root row past its rows).  Median of
`--steps` calls after `--warmup`.  On a 32-query sample every entry point's rows are checked against pyhybrid over the
shim's lists.  Prints the card and its power limit, then one JSON line per (pairing, batch).

    python tools/bench_hybrid_sharded.py [--rows 1000000] [--shards 2] [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosdata_b200 as cdb  # noqa: E402
from cosdata_b200.sharding import ShardGroup, shard_range  # noqa: E402
from tests import pyhybrid as ph  # noqa: E402
from tests.sparse_data import concat_csr, slice_csr, zipf_csr  # noqa: E402
from tests.tfidf_data import zipf_docs, zipf_queries  # noqa: E402

CHUNK = 500_000
DIM = 768
TOP_K = 10
DENSE = {"mode": cdb.SearchMode.HNSW, "ef_search": 128, "shortlist_size": 64}
PAIRS = [("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf")]
HN_GAP = 1 << 21


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def build_group(devs, bounds, sp_corpus, tf_corpus):
    g, keep = ShardGroup.local(devs), []
    for r, dev in enumerate(devs):
        b0, b1 = bounds[r], bounds[r + 1]
        # the graph build keeps one more row for its root: dense shards' id ranges are spaced HN_GAP apart
        d = cdb.DenseIndex(dim=DIM, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=b1 - b0 + 1, keep_raw_f32=True,
                           id_base=r * HN_GAP, device=dev)
        d.append_synthetic(11, b1 - b0, b0)
        d.build_graph(9, 32, 64, 128, 64, 4096, 7)
        part = slice_csr(sp_corpus, b0, b1)
        sp = cdb.SparseIndex(quantization_bits=4, values_upper_bound=3.0, capacity_rows=b1 - b0, capacity_pairs=len(part[1]) + 8,
                             id_base=b0, device=dev)
        sp.append(part)
        part = slice_csr(tf_corpus, b0, b1)
        tf = cdb.TfIdfIndex(capacity_rows=b1 - b0, capacity_pairs=len(part[1]) + 8, id_base=b0, device=dev)
        tf.append(part, 1)
        g.attach(r, d)
        g.attach_sparse(r, sp)
        g.attach_tfidf(r, tf)
        keep += [d, sp, tf]
    return g, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parity-queries", type=int, default=32)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    dev = torch.device("cuda", 0)
    name = card()
    print(json.dumps({"card": name, "gpus": cdb.device_count()}), flush=True)
    n, w = a.rows, a.shards
    t0 = time.perf_counter()
    sp_corpus = concat_csr([zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))])
    tf_corpus = concat_csr([zipf_docs(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))])
    devs = list(range(w)) if cdb.device_count() >= w else [0] * w
    groups = {w: build_group(devs, [shard_range(n, w, r)[0] for r in range(w)] + [n], sp_corpus, tf_corpus),
              1: build_group([0], [0, n], sp_corpus, tf_corpus)}
    del sp_corpus, tf_corpus
    torch.cuda.synchronize()
    print(json.dumps({"setup_s": round(time.perf_counter() - t0, 1), "rows": n, "shards": w, "loopback": devs.count(0) > 1}), flush=True)

    dq_all = cdb.synth_matrix(12, 1024, DIM)
    sq_all = zipf_csr(7, 1024, mean_pairs=40)
    tq_all = zipf_queries(7, 1024, vocab=1_000_000)
    k3 = 3 * TOP_K
    s = torch.cuda.Stream(dev)

    def t(x):
        x = np.ascontiguousarray(x)
        return torch.from_numpy(x.view({np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(x.dtype, x.dtype))).to(dev)

    def host_timed(fn):
        for _ in range(a.warmup):
            fn()
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            out = fn()
            ts.append(1e3 * (time.perf_counter() - t0))
        return float(np.median(ts)), out

    def dev_timed(fn):
        for _ in range(a.warmup):
            fn()
        s.synchronize()
        ts = []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            fn()
            e1.record(s)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    for pair in PAIRS:
        for b in (1, 64, 1024):
            dq, sq, tq = dq_all[:b], slice_csr(sq_all, 0, b), tq_all[:b]
            sp_opts = cdb.SparseSearchOptions(0, 0.0)
            kw = {"dense": (dq, DENSE), "sparse": (sq, sp_opts), "tfidf": tq}
            kw = {p: kw[p] for p in pair}
            res = {"pair": "+".join(pair), "batch": b, "top_k": TOP_K, "card": name}
            sel = np.arange(0, b, max(1, b // a.parity_queries))[: a.parity_queries]
            parity = True
            for gw, (g, _) in groups.items():
                run = {"dense": lambda g=g: g.search(dq, k3, **DENSE)[:3],
                       "sparse": lambda g=g: g.search_sparse(sq, cdb.SparseSearchOptions(k3, 0.0)),
                       "tfidf": lambda g=g: g.search_tfidf(tq, k3)}

                def shim(g=g, run=run):
                    la, lb = run[pair[0]](), run[pair[1]]()
                    return cdb.rrf_fuse(la[0], la[2], lb[0], lb[2], 60.0)

                res[f"g{gw}_entry_ms"], got = host_timed(lambda g=g: g.hybrid_search(TOP_K, 60.0, **kw))
                res[f"g{gw}_shim_ms"], via = host_timed(shim)
                la, lb = run[pair[0]](), run[pair[1]]()
                want = ph.fuse_batch(la[0][sel], la[2][sel], lb[0][sel], lb[2][sel], 60.0, ld_out=6 * TOP_K)
                for x in (got, via):
                    parity &= bool(np.array_equal(x[2][sel], want[2]) and np.array_equal(x[0][sel][:, :6 * TOP_K], want[0])
                                   and np.array_equal(x[1][sel][:, :6 * TOP_K].view(np.uint32), want[1].view(np.uint32)))
                if gw == 1 and "tfidf" not in pair:
                    ids = torch.zeros((b, 6 * TOP_K), dtype=torch.int32, device=dev)
                    sc = torch.zeros((b, 6 * TOP_K), dtype=torch.float32, device=dev)
                    ct = torch.zeros(b, dtype=torch.int32, device=dev)
                    d_q, d_s = t(dq), [t(x) for x in sq]
                    dkw = {"dense": (d_q.data_ptr(), DENSE), "sparse": (tuple(x.data_ptr() for x in d_s), sp_opts)}
                    res["g1_device_ms"] = round(dev_timed(lambda: g.hybrid_search_device(
                        b, ids.data_ptr(), sc.data_ptr(), ct.data_ptr(), None, s.cuda_stream, TOP_K, 60.0, **dkw)), 4)
                    s.synchronize()
                    dev_got = (ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), ct.cpu().numpy().view(np.uint32))
                    parity &= bool(all(np.array_equal(np.asarray(x)[sel].view(np.uint32), np.asarray(y)[sel].view(np.uint32))
                                       for x, y in zip(dev_got, got[:3])))
            for key in list(res):
                if key.endswith("_ms"):
                    res[key] = round(res[key], 4)
            res[f"parity_{sel.size}q"] = parity
            print(json.dumps(res), flush=True)
    for g, keep in groups.values():
        g.close()
        for x in keep:
            x.close()


if __name__ == "__main__":
    main()
