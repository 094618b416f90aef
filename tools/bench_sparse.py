"""Sparse inverted index on one GPU: append time, QPS at batch 1 / 64 / 1024 with and without the raw-value re-rank, and
posting-entry bytes visited over device time, on a seeded SPLADE-like corpus (vocabulary 30522, Zipf dim popularity,
~120 pairs per row, ~40 per query).  At the smallest size it also times the CPU oracle on all host threads over a query
sample and checks the GPU results against it.  Prints one JSON line per corpus size.

    python tools/bench_sparse.py [--rows 1000000,8800000] [--steps 5]
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
from tests import pysparse as ps  # noqa: E402
from tests.sparse_data import concat_csr, slice_csr, zipf_csr  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data sheet
CHUNK = 500_000     # rows generated and appended per call


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def entries_visited(df, queries):
    """posting entries the default threshold (0.0: every key of every query dim) reads, summed over the queries"""
    return int(df[queries[1]].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1000000,8800000")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--oracle-queries", type=int, default=64)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    dev = torch.device("cuda", 0)
    name = card()
    ub = 3.0
    for n in [int(x) for x in a.rows.split(",")]:
        chunks = [zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))]
        pairs = sum(len(c[1]) for c in chunks)
        ix = cdb.SparseIndex(quantization_bits=4, values_upper_bound=ub, capacity_rows=n, capacity_pairs=pairs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in chunks:
            ix.append(c)
        torch.cuda.synchronize()
        append_s = time.perf_counter() - t0
        df = np.zeros(30522, np.int64)
        for c in chunks:
            df += np.bincount(c[1], minlength=30522)
        queries = zipf_csr(7, 1024, mean_pairs=40)
        res = dict(rows=n, pairs=pairs, card=name, append_s=round(append_s, 3))
        for rerank in (False, True):
            opts = cdb.SparseSearchOptions(10, 0.0, rerank, 5)
            p = opts.params()
            for b in (1, 64, 1024):
                q = slice_csr(queries, 0, b)
                o, d, v = [torch.from_numpy(x.astype(t)).to(dev) for x, t in zip(q, (np.int64, np.int32, np.float32))]
                ids = torch.zeros((b, 10), dtype=torch.int32, device=dev)
                sc = torch.zeros((b, 10), dtype=torch.float32, device=dev)
                cnt = torch.zeros(b, dtype=torch.int32, device=dev)
                s = torch.cuda.current_stream(dev)

                def call():
                    rc = _lib.load().cdb_sparse_search_batch_device(ix.h, o.data_ptr(), d.data_ptr(), v.data_ptr(), b, C.byref(p),
                                                                    ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), C.c_void_p(s.cuda_stream))
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
                byts = entries_visited(df, q) * 4
                tag = f"{'rerank' if rerank else 'plain'}_b{b}"
                res[f"qps_{tag}"] = round(b / (ms / 1e3), 1)
                res[f"ms_{tag}"] = round(ms, 3)
                res[f"entry_GBps_{tag}"] = round(byts / (ms / 1e3) / 1e9, 1)
                res[f"entry_share_of_hbm_{tag}"] = round(byts / (ms / 1e3) / HBM_BPS, 3)
        if n <= 1_000_000:
            corpus = concat_csr(chunks)
            sample = np.arange(0, 1024, 1024 // a.oracle_queries)
            sub = concat_csr([slice_csr(queries, int(i), int(i) + 1) for i in sample])
            for rerank in (False, True):
                t0 = time.perf_counter()
                want = ps.search(corpus, sub, 10, bits=4, ub=ub, rerank=rerank, factor=5)
                cpu_s = time.perf_counter() - t0
                got = ix.batch_search(queries, cdb.SparseSearchOptions(10, 0.0, rerank, 5))
                ok = (np.array_equal(got[0][sample], want[0]) and np.array_equal(got[2][sample], want[2])
                      and np.array_equal(got[1][sample].view(np.uint32), want[1].view(np.uint32)))
                tag = "rerank" if rerank else "plain"
                res[f"oracle_qps_{tag}_{os.cpu_count()}threads_incl_list_build"] = round(len(sample) / cpu_s, 2)
                res[f"parity_{tag}_{len(sample)}q"] = bool(ok)
        ix.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
