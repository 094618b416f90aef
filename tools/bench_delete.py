"""Cost of deleting rows from an HNSW graph on the GPU (cdb_index_delete_rows) and the recall that remains.

On clustered rows from bench.py's c3 generator (f16 storage, cosine, the reference defaults: 9 levels, 32/64 neighbours,
ef_construction 128, shortlist 64), one build of N rows, then
  (a) `--single` rows deleted one call at a time with max_batch = 1 (per-call times);
  (b) 0.01 N rows deleted in one batched call, then (c) 0.1 N rows more in one batched call;
and recall@10 (ef_search 128, 1024 queries) after (c), against the exact scan over the live rows, next to a fresh build over
the live rows.  Times are host clocks around calls that end in a device synchronise.  Prints one JSON line with the card
name and power limit.

    python tools/bench_delete.py [--rows 1000000] [--dim 768] [--single 1000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_insert import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--single", type=int, default=1000)
    ap.add_argument("--queries", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb

    N, D, B, k = args.rows, args.dim, args.queries, 10
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

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    rec = {"card": card(), "rows": N, "dim": D, "storage": "f16", "metric": "cosine",
           "params": {"num_levels": 9, "neighbors": [32, 64], "ef_construction": 128, "shortlist": 64, "ef_delete": 512},
           "times_s": {}, "recall_at_10": {}}
    ix = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 1, keep_raw_f32=True)
    ix.append_device(X.data_ptr(), N)
    t, _ = timed(lambda: ix.build_graph(9, 32, 64, 128, 64, 4096, 7))
    rec["times_s"]["build"] = t
    order = np.random.default_rng(5).permutation(N).astype(np.uint32)
    s1, s2 = args.single, args.single + N // 100
    s3 = s2 + N // 10
    per = []
    for r in order[:s1]:
        t, st = timed(lambda: ix.delete_rows([r], 64, 1))
        per.append(t)
        assert st[0] != 1
    rec["times_s"]["a_single_total"] = float(np.sum(per))
    rec["times_s"]["a_single_mean"] = float(np.mean(per))
    rec["times_s"]["a_single_max"] = float(np.max(per))
    t, st = timed(lambda: ix.delete_rows(order[s1:s2]))
    rec["times_s"][f"b_batched_{s2 - s1}"] = t
    t, st = timed(lambda: ix.delete_rows(order[s2:s3]))
    rec["times_s"][f"c_batched_{s3 - s2}"] = t
    rec["status_2"] = int((st == 2).sum())
    live = np.sort(order[s3:])
    ids, _, _, _ = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=128, shortlist_size=64)
    root = N   # the exact scan skips deleted rows but sees the root row, which HNSW results never contain

    def hits(res, want):
        return sum(len(set(int(x) for x in res[i]) & set(want[i])) for i in range(B)) / (B * k)

    gk, _, _, _ = ix.batch_search(queries, k + 1, cdb.SearchMode.BRUTE_RAW, exact_only=True)
    want = [[int(x) for x in gk[i] if int(x) != root][:k] for i in range(B)]
    rec["recall_at_10"]["after_deletes"] = hits(ids, want)
    ix.close()
    fresh = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=live.size + 1, keep_raw_f32=True)
    Xl = X[torch.from_numpy(live.astype(np.int64)).to(dev)].contiguous()
    torch.cuda.synchronize()   # the index copies on its own stream
    fresh.append_device(Xl.data_ptr(), live.size)
    t, _ = timed(lambda: fresh.build_graph(9, 32, 64, 128, 64, 4096, 7))
    rec["times_s"]["fresh_build_live"] = t
    fi, _, _, _ = fresh.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=128, shortlist_size=64)
    fi = np.where(fi < live.size, live[np.minimum(fi, live.size - 1)], 0xFFFFFFFF)
    rec["recall_at_10"]["fresh_build_live"] = hits(fi, want)
    fresh.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
