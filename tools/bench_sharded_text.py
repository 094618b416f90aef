"""Sharded sparse and TF-IDF search against one index over the same corpus: host-form call time (queries in, results out,
median of --steps calls after one warm-up) at batch 1 / 64 / 1024, sparse with and without the raw-value re-rank (top 10,
factor 5) and TF-IDF (top 10), plus a parity check of every batch (ids, counts and score bits of the group against the
single index).  TF-IDF also times the device form (cdb_tfidf_search_batch_sharded_device: queries and results in device
memory, the group's idf summed on the device) by CUDA events over --steps calls on one stream, next to the host form, on
the --shards group and on a one-slot group holding the whole index, and checks its results against the host form's.  Corpora: the 1M-row corpora of tools/bench_sparse.py and tools/bench_tfidf.py, split into --shards
contiguous id ranges.  With one GPU the shards share it and the gathers are device copies (loopback), so the numbers are
the protocol's overhead on one card, not scaling; with as many GPUs as shards each shard has its own card and NCCL.
Prints the card and its power limit, then one JSON line per workload.

    python tools/bench_sharded_text.py [--rows 1000000] [--shards 2] [--steps 10]
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
from tests.sparse_data import concat_csr, slice_csr, zipf_csr  # noqa: E402
from tests.tfidf_data import query_csr, zipf_docs, zipf_queries  # noqa: E402

CHUNK = 500_000
VOCAB_TFIDF = 1_000_000


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, steps):
    fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def same(a, b):
    return (np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
            and np.array_equal(np.ascontiguousarray(a[1]).view(np.uint32), np.ascontiguousarray(b[1]).view(np.uint32)))


def device_form(g, qs, k, steps):
    """(ms per call by CUDA events, results) of the group's device-form TF-IDF search on one torch stream"""
    import torch
    dev = torch.device("cuda", 0)
    o, h = query_csr(qs)
    d_o = torch.from_numpy(o.astype(np.int64)).to(dev)
    d_h = torch.from_numpy(h.view(np.int32)).to(dev)
    nq = len(qs)
    ids = torch.zeros((nq, k), dtype=torch.int32, device=dev)
    sc = torch.zeros((nq, k), dtype=torch.float32, device=dev)
    ct = torch.zeros(nq, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream(dev)

    def call():
        g.search_tfidf_device(d_o.data_ptr(), d_h.data_ptr(), nq, int(h.size), k, ids.data_ptr(), sc.data_ptr(), ct.data_ptr(),
                              s.cuda_stream)
    call()
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(steps):
        call()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps, (ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), ct.cpu().numpy().view(np.uint32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    import torch  # noqa: F401  before the library can load a system libnccl.so.2 that torch's CUDA library cannot share
    assert cdb.device_count() > 0, "needs a CUDA device"
    n, w = a.rows, a.shards
    devs = list(range(w)) if cdb.device_count() >= w else [0] * w
    mode = "nccl" if len(set(devs)) == w else "loopback_one_gpu_protocol_overhead"
    name = card()
    print(json.dumps({"card": name, "shards": w, "devices": devs, "mode": mode}), flush=True)
    bounds = [shard_range(n, w, r)[0] for r in range(w)] + [n]

    # sparse: bench_sparse.py's corpus (vocabulary 30522, ~120 pairs per row, ~40 per query), values_upper_bound 3.0
    corpus = concat_csr([zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))])
    queries = zipf_csr(7, 1024, mean_pairs=40)
    whole = cdb.SparseIndex(quantization_bits=4, values_upper_bound=3.0, capacity_rows=n, capacity_pairs=len(corpus[1]))
    whole.append(corpus)
    g = ShardGroup.local(devs)
    parts = []
    for r in range(w):
        piece = slice_csr(corpus, bounds[r], bounds[r + 1])
        ix = cdb.SparseIndex(quantization_bits=4, values_upper_bound=3.0, capacity_rows=bounds[r + 1] - bounds[r],
                             capacity_pairs=len(piece[1]) + 1, id_base=bounds[r], device=devs[r])
        ix.append(piece)
        g.attach_sparse(r, ix)
        parts.append(ix)
    for rerank in (False, True):
        opts = cdb.SparseSearchOptions(10, 0.0, rerank, 5)
        for b in (1, 64, 1024):
            q = slice_csr(queries, 0, b)
            single = timed(lambda: whole.batch_search(q, opts), a.steps)
            sharded = timed(lambda: g.search_sparse(q, opts), a.steps)
            res = dict(workload=f"sparse_{'rerank_f5' if rerank else 'plain'}", rows=n, batch=b, top_k=10, mode=mode, card=name,
                       single_ms=round(single, 3), sharded_ms=round(sharded, 3), sharded_over_single=round(sharded / single, 3),
                       parity=bool(same(g.search_sparse(q, opts), whole.batch_search(q, opts))))
            print(json.dumps(res), flush=True)
    g.close()
    for x in parts + [whole]:
        x.close()
    del corpus

    # TF-IDF: bench_tfidf.py's corpus (vocabulary 1M, ~40 terms per document, 3..12 terms per query)
    docs = concat_csr([zipf_docs(1000 + i, min(CHUNK, n - r0), vocab=VOCAB_TFIDF) for i, r0 in enumerate(range(0, n, CHUNK))])
    tq = zipf_queries(7, 1024, vocab=VOCAB_TFIDF)
    whole = cdb.TfIdfIndex(capacity_rows=n, capacity_pairs=len(docs[1]))
    whole.append(docs, 1)
    g = ShardGroup.local(devs)
    parts = []
    for r in range(w):
        piece = slice_csr(docs, bounds[r], bounds[r + 1])
        ix = cdb.TfIdfIndex(capacity_rows=bounds[r + 1] - bounds[r], capacity_pairs=len(piece[1]) + 1, id_base=bounds[r], device=devs[r])
        ix.append(piece, 1)
        g.attach_tfidf(r, ix)
        parts.append(ix)
    one = ShardGroup.local([0])
    one.attach_tfidf(0, whole)
    for b in (1, 64, 1024):
        q = tq[:b]
        single = timed(lambda: whole.batch_search(q, 10), a.steps)
        sharded = timed(lambda: g.search_tfidf(q, 10), a.steps)
        res = dict(workload="tfidf", rows=n, batch=b, top_k=10, mode=mode, card=name, single_ms=round(single, 3),
                   sharded_ms=round(sharded, 3), sharded_over_single=round(sharded / single, 3),
                   parity=bool(same(g.search_tfidf(q, 10), whole.batch_search(q, 10))))
        print(json.dumps(res), flush=True)
        for label, grp in ((f"{w}_slots_{mode}", g), ("1_slot", one)):
            host = timed(lambda: grp.search_tfidf(q, 10), a.steps)
            dev_ms, got = device_form(grp, q, 10, a.steps)
            res = dict(workload="tfidf_device_form", group=label, rows=n, batch=b, top_k=10, card=name, host_form_ms=round(host, 3),
                       device_form_event_ms=round(dev_ms, 3), parity_with_host_form=bool(same(got, grp.search_tfidf(q, 10))))
            print(json.dumps(res), flush=True)
    one.close()
    g.close()
    for x in parts + [whole]:
        x.close()


if __name__ == "__main__":
    main()
