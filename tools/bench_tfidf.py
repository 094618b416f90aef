"""TF-IDF / BM25 index on one GPU: append time, the idf refresh that every append and delete ends with, and queries/s at
batch 1 / 64 / 1024 (CUDA events around the whole device search), with posting bytes visited over that time, on a seeded
Zipf corpus (~40 terms per document, vocabulary 1M hashes, queries of 3-12 terms, tf from bm25_term_frequency).  Over a
query sample it times the CPU oracle, checks GPU-oracle parity (the `query` summation order) and counts the ids whose score
differs between the `query` order and the reference's heap order.  Prints the card and its power limit, then one JSON line
per corpus size.

    python tools/bench_tfidf.py [--rows 1000000,8800000] [--steps 5] [--oracle-queries 32]
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
from tests import pytfidf as pt  # noqa: E402
from tests.sparse_data import concat_csr  # noqa: E402
from tests.tfidf_data import query_csr, zipf_docs, zipf_queries  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data sheet
CHUNK = 500_000     # documents generated and appended per call
VOCAB = 1_000_000


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1000000,8800000")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--oracle-queries", type=int, default=32)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    dev = torch.device("cuda", 0)
    name = card()
    print(json.dumps({"card": name}), flush=True)
    queries = zipf_queries(7, 1024, vocab=VOCAB)
    for n in [int(x) for x in a.rows.split(",")]:
        chunks = [zipf_docs(1000 + i, min(CHUNK, n - r0), vocab=VOCAB) for i, r0 in enumerate(range(0, n, CHUNK))]
        pairs = sum(len(c[1]) for c in chunks)
        ix = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=pairs + 64)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in chunks:
            ix.append(c, 1)
        torch.cuda.synchronize()
        append_s = time.perf_counter() - t0
        # df per hash from the data: the posting entries a query visits
        uh, cnt = np.unique(np.concatenate([c[1] for c in chunks]), return_counts=True)
        n_terms = int(uh.size)
        res = dict(rows=n, pairs=pairs, terms=n_terms, card=name, append_s=round(append_s, 3),
                   append_chunk_rows=CHUNK)
        # the idf refresh: a one-row delete is a gather of its terms plus the refresh of every idf; a one-row append also
        # rebuilds the last partial tile
        ts = []
        for r in range(5):
            t0 = time.perf_counter()
            ix.delete_embedding([r * 7919 % n], 2)
            ts.append(time.perf_counter() - t0)
        res["delete_1row_ms"] = round(1e3 * float(np.median(ts)), 3)
        one = (np.array([0, 1], np.uint64), np.array([uh[0]], np.uint32), np.array([1.0], np.float32))
        t0 = time.perf_counter()
        ix.append(one, 2)
        res["append_1row_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
        for b in (1, 64, 1024):
            qo, qh = query_csr(queries[:b])
            o = torch.from_numpy(qo.astype(np.int64)).to(dev)
            h = torch.from_numpy(qh.astype(np.int32)).to(dev)
            ids = torch.zeros((b, 10), dtype=torch.int32, device=dev)
            sc = torch.zeros((b, 10), dtype=torch.float32, device=dev)
            ct = torch.zeros(b, dtype=torch.int32, device=dev)
            s = torch.cuda.current_stream(dev)

            def call():
                rc = _lib.load().cdb_tfidf_search_batch_device(ix.h, o.data_ptr(), h.data_ptr(), b, 10, ids.data_ptr(), sc.data_ptr(),
                                                                ct.data_ptr(), C.c_void_p(s.cuda_stream))
                assert rc == 0
            call()
            s.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(a.steps):
                call()
            e1.record(s)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
            pos = np.searchsorted(uh, qh)
            hit = (pos < uh.size) & (uh[np.minimum(pos, uh.size - 1)] == qh)
            byts = int(cnt[pos[hit]].sum()) * 8          # (row, tf) entries of 8 bytes
            res[f"qps_b{b}"] = round(b / (ms / 1e3), 1)
            res[f"ms_b{b}"] = round(ms, 3)
            res[f"entry_GBps_b{b}"] = round(byts / (ms / 1e3) / 1e9, 1)
            res[f"entry_share_of_hbm_b{b}"] = round(byts / (ms / 1e3) / HBM_BPS, 3)
        if n <= 1_000_000:
            corpus = concat_csr(chunks)
            orc = pt.Oracle()
            orc.append(corpus, 1)
            for r in range(5):
                orc.delete([r * 7919 % n], 2)
            orc.append(one, 2)
            sample = np.arange(0, 1024, 1024 // a.oracle_queries)
            sub = [queries[int(i)] for i in sample]
            t0 = time.perf_counter()
            want = orc.search(query_csr(sub), 10)
            cpu_s = time.perf_counter() - t0
            got = ix.batch_search(queries, 10)
            ok = (np.array_equal(got[0][sample], want[0]) and np.array_equal(got[2][sample], want[2])
                  and np.array_equal(got[1][sample].view(np.uint32), want[1].view(np.uint32)))
            res[f"oracle_qps_{os.cpu_count()}threads"] = round(len(sample) / cpu_s, 2)
            res[f"parity_{len(sample)}q"] = bool(ok)
            differ = touched = 0
            for q in sub:
                sa, ta, _, _, _ = orc.scores(q, "query")
                sb, _, _, _, pb = orc.scores(q, "heap")
                touched += int(ta.sum())
                differ += int((ta & (sa.view(np.uint32) != sb.view(np.uint32))).sum())
            top_differ = sum(not np.array_equal(x, y) for x, y in
                             zip(want[0], orc.search(query_csr(sub), 10, "heap")[0]))
            res["heap_vs_query_ids_differing"] = differ
            res["heap_vs_query_ids_scored"] = touched
            res["heap_vs_query_top10_lists_differing"] = int(top_differ)
            orc.close()
        ix.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
