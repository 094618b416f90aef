"""Sparse search with top_k None (every candidate, cdb_sparse_search_batch_all) on one GPU, on the 1M-row corpus of
tools/bench_sparse.py (vocabulary 30522, Zipf dim popularity, ~120 pairs per row, ~40 per query, 4 bits, values_upper_bound
3.0).  For batch 1 and 16, thresholds 0.0 and 0.5, with and without re-rank: median ms per call (with min and max) and
queries/s (host query arrays in, every result read out into numpy), candidates per query and per second, result bytes,
and the share of the call the device-to-host copies take (torch.profiler over one call, with its per-kernel times).  Checks a query sample against the CPU oracle
(tests/sparse_oracle.c, k = n_rows, factor 1) and times that oracle.  Prints the card and one JSON line.

    python tools/bench_sparse_all.py [--rows 1000000] [--steps 7]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosdata_b200 as cdb  # noqa: E402
from tests import pysparse as ps  # noqa: E402
from tests.sparse_data import concat_csr, slice_csr, zipf_csr  # noqa: E402

CHUNK = 500_000     # rows generated and appended per call, as tools/bench_sparse.py


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def profile_call(call):
    """device-to-host copy time and per-kernel time (ms) of one call, from torch.profiler's CUDA activities"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        call()
    dtoh, kernels = 0.0, {}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3
        if not t:
            continue
        if "Memcpy DtoH" in e.key:
            dtoh += t
        elif "Memcpy" not in e.key and "Memset" not in e.key:
            m = re.search(r"(sp_\w+|Device\w+)", e.key)
            name = m.group(1) if m else e.key[:40]
            kernels[name] = round(kernels.get(name, 0.0) + t, 3)
    return dtoh, kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--oracle-sample", default="0,3")
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    name = card()
    n, ub = a.rows, 3.0
    chunks = [zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))]
    pairs = sum(len(c[1]) for c in chunks)
    ix = cdb.SparseIndex(quantization_bits=4, values_upper_bound=ub, capacity_rows=n, capacity_pairs=pairs)
    for c in chunks:
        ix.append(c)
    queries = zipf_csr(7, 1024, mean_pairs=40)
    res = dict(card=name, rows=n, pairs=pairs, steps=a.steps)
    for thr in (0.0, 0.5):
        for rerank in (False, True):
            opts = cdb.SparseSearchOptions(None, thr, rerank)
            for b in (1, 16):
                q = slice_csr(queries, 0, b)
                call = lambda: ix.batch_search_all(q, opts)   # noqa: E731
                off, _, _ = call()                             # warm-up
                torch.cuda.synchronize()
                times = []
                for _ in range(a.steps):                       # each call ends with its results in host memory
                    t0 = time.perf_counter()
                    off, _, _ = call()
                    times.append((time.perf_counter() - t0) * 1e3)
                ms = float(np.median(times))
                total = int(off[-1])
                dtoh, kernels = profile_call(call)
                tag = f"thr{thr}_{'rerank' if rerank else 'plain'}_b{b}"
                res[tag] = dict(ms=round(ms, 3), ms_min=round(min(times), 3), ms_max=round(max(times), 3),
                                qps=round(b / (ms / 1e3), 1), cand_per_query=round(total / b), cand_per_s=round(total / (ms / 1e3)), result_bytes=total * 8 + (b + 1) * 8,
                                dtoh_ms=round(dtoh, 3), dtoh_share=round(dtoh / ms, 3) if dtoh else None, kernel_ms=kernels)
                print(tag, json.dumps(res[tag]), flush=True)
    corpus = concat_csr(chunks)
    sample = [int(x) for x in a.oracle_sample.split(",")]
    sub = concat_csr([slice_csr(queries, i, i + 1) for i in sample])
    t0 = time.perf_counter()
    ps.search(corpus, slice_csr(queries, 0, 0), 1, bits=4, ub=ub)     # no query: the oracle's list build alone
    res["oracle_list_build_s"] = round(time.perf_counter() - t0, 2)
    for rerank in (False, True):
        opts = cdb.SparseSearchOptions(None, 0.0, rerank)
        t0 = time.perf_counter()
        w_ids, w_scores, w_counts = ps.search(corpus, sub, n, bits=4, ub=ub, rerank=rerank, factor=1)
        cpu_s = time.perf_counter() - t0
        off, ids, scores = ix.batch_search_all(slice_csr(queries, 0, max(sample) + 1), opts)
        ok = True
        for i, qq in enumerate(sample):
            b, e, c = int(off[qq]), int(off[qq + 1]), int(w_counts[i])
            ok &= e - b == c and np.array_equal(ids[b:e], w_ids[i, :c]) and np.array_equal(scores[b:e].view(np.uint32),
                                                                                         w_scores[i, :c].view(np.uint32))
        tag = "rerank" if rerank else "plain"
        res[f"oracle_s_{tag}_{len(sample)}q_{os.cpu_count()}threads_incl_list_build"] = round(cpu_s, 2)
        res[f"parity_{tag}_{len(sample)}q"] = bool(ok)
    ix.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
