"""Cost of growing an HNSW graph on the GPU (cdb_index_insert_graph) against building it in one go.

On clustered rows from bench.py's c3 generator (f16 storage, cosine, the reference defaults: 9 levels, 32/64 neighbours,
ef_construction 128), this measures
  (a) a one-shot build of N rows;
  (b) a build of 0.9 N rows + one insert of 0.1 N rows;
  (c) a build of 0.9 N rows + `--calls` inserts of 0.1 N / calls rows each (per-call times: the cost of a call must not grow
      with the number of calls beyond the geometric growth of the level arrays);
  (d) the slot-state derivation of the uploaded 0.9 N graph (hnsw_slot_state_kernel, via the first
      cdb_index_read_graph_slot_scores; the second call, which only copies, is reported next to it);
and recall@10 (ef_search 128, 1024 queries, against the exact scan of the same index) of (a), (b) and (c).  Times are host
clocks around calls that end in a device synchronise.  Prints one JSON line with the card name and power limit.

    python tools/bench_insert.py [--rows 1000000] [--dim 768] [--calls 100]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--queries", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb

    N, D, B, k = args.rows, args.dim, args.queries, 10
    n0 = N - N // 10
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    g = torch.Generator(device=dev)           # bench.py's c3 generator
    g.manual_seed(1234)
    ncent = 4096
    centres = torch.randn((ncent, D), generator=g, device=dev)
    scale = 1.0 / (4.5 * 1.06)

    def draw(m):
        idx = torch.randint(0, ncent, (m,), generator=g, device=dev)
        return ((centres[idx] + 0.35 * torch.randn((m, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()

    X = torch.cat([draw(min(500_000, N - o)) for o in range(0, N, 500_000)])
    queries = draw(B).cpu().numpy()
    torch.cuda.synchronize()
    ST, MK = cdb.StorageType.HalfPrecisionFP, cdb.DistanceMetricKind.Cosine

    def index(rows):
        ix = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 1, keep_raw_f32=True)
        ix.append_device(X[:rows].data_ptr(), rows)
        return ix

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def recall(ix):   # the exact scan also sees the root row, which the HNSW results never contain
        ids, _, _, _ = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=128, shortlist_size=64)
        gt, _, _, _ = ix.batch_search(queries, k + 1, cdb.SearchMode.BRUTE_RAW, exact_only=True)
        hits = 0
        for i in range(B):
            want = [int(x) for x in gt[i] if int(x) != root_row[0]][:k]
            hits += len(set(int(x) for x in ids[i]) & set(want))
        return hits / (B * k)

    def append(ix, a, b):
        ix.append_device(X[a:b].data_ptr(), b - a)

    rec = {"card": card(), "rows": N, "dim": D, "storage": "f16", "metric": "cosine",
           "params": {"num_levels": 9, "neighbors": [32, 64], "ef_construction": 128}, "times_s": {}, "recall_at_10": {}}
    root_row = [N]
    # (a) one-shot build
    ix = index(N)
    t, _ = timed(lambda: ix.build_graph(9, 32, 64, 128, 64, 4096, 7))
    rec["times_s"]["a_build_all"] = t
    root_row[0] = N
    rec["recall_at_10"]["a"] = recall(ix)
    ix.close()
    # (b) build 0.9 N + one insert of 0.1 N; (d) slot state of the uploaded 0.9 N graph
    ix = index(n0)
    t, _ = timed(lambda: ix.build_graph(9, 32, 64, 128, 64, 4096, 7))
    rec["times_s"]["b_build_0.9"] = t
    g0 = ix.read_graph()
    codes, mags = ix.read_codes(0, n0 + 1)
    up = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=n0 + 1)
    up.append_codes(codes, mags)
    up.set_graph(9, 32, 64, g0["entry"], g0["root_row"], g0["node_row"], g0["adj"], g0["child"])
    t1, _ = timed(up.read_graph_slot_scores)
    t2, _ = timed(up.read_graph_slot_scores)
    rec["times_s"]["d_slot_state_first_read"] = t1
    rec["times_s"]["d_slot_state_copy_only_read"] = t2
    up.close()
    del g0, codes, mags
    append(ix, n0, N)
    t, failed = timed(lambda: ix.insert_graph(128, 64, 4096, 7))
    rec["times_s"]["b_insert_0.1"] = t
    rec["b_failed"] = int(failed.sum())
    root_row[0] = n0
    rec["recall_at_10"]["b"] = recall(ix)
    ix.close()
    # (c) build 0.9 N + `calls` inserts
    ix = index(n0)
    t, _ = timed(lambda: ix.build_graph(9, 32, 64, 128, 64, 4096, 7))
    rec["times_s"]["c_build_0.9"] = t
    per = []
    step = (N - n0) // args.calls
    for c in range(args.calls):
        a = n0 + c * step
        b = N if c == args.calls - 1 else a + step
        append(ix, a, b)
        t, _ = timed(lambda: ix.insert_graph(128, 64, 4096, 7))
        per.append(t)
    rec["times_s"]["c_inserts_total"] = float(np.sum(per))
    rec["times_s"]["c_insert_first10_mean"] = float(np.mean(per[:10]))
    rec["times_s"]["c_insert_last10_mean"] = float(np.mean(per[-10:]))
    rec["times_s"]["c_insert_max"] = float(np.max(per))
    rec["recall_at_10"]["c"] = recall(ix)
    ix.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
