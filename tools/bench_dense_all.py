"""Dense HNSW search without top_k (CDB_SEARCH_ALL_CANDIDATES) against top_k = 10, and the filtered sharded search.

1. HNSW: N rows (default 1M) of bench.py's clustered c3 rows, 768-dim f16 storage with raw f32 rows kept, cosine, graph built
   on the GPU (9 levels, 32/64 neighbours, ef_construction 128).  ef 128; batches of 1, 64 and 1024 queries; top_k None (row
   width (num_levels + 1) * 100) against k = 10, both through cdb_search_batch_device on one stream, ms per call from CUDA
   events (median after warm-up).  The None rows' first 10 columns are not compared with k = 10: the top-k search re-ranks
   only the best 5 * k candidates of the traversal.
2. Filtered sharded search: a loopback group of 2 replica-graph shards on one GPU (tests/mdgraph.py graphs, 3000 embeddings
   each, 128-dim f16), k = 10, one filter per query for three of four queries, batch 1024: cdb_search_batch_filtered_sharded
   against the two per-shard cdb_search_batch_filtered calls plus the numpy merge (sharding.merge_packed), host clock around
   each synchronising call; the two results are compared.
Prints a table and one JSON line with the card name and power limit read in the same run.

    python tools/bench_dense_all.py [--rows 1000000] [--dim 768]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_insert_replicas import card  # noqa: E402


def hnsw_part(args, rec):
    import torch
    import cosdata_b200 as cdb

    N, D, ef, LEVELS = args.rows, args.dim, 128, 9
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)           # bench.py's c3 generator
    g.manual_seed(1234)
    ncent = 4096
    centres = torch.randn((ncent, D), generator=g, device=dev)
    scale = 1.0 / (4.5 * 1.06)

    def draw(m):
        idx = torch.randint(0, ncent, (m,), generator=g, device=dev)
        return ((centres[idx] + 0.35 * torch.randn((m, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()

    X = torch.cat([draw(min(500_000, N - o)) for o in range(0, N, 500_000)])
    Q = draw(1024)
    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.HalfPrecisionFP, metric=cdb.DistanceMetricKind.Cosine, capacity=N + 1,
                        keep_raw_f32=True)
    ix.append_device(X.data_ptr(), N)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ix.build_graph(LEVELS, 32, 64, 128, 64, 4096, 1)
    torch.cuda.synchronize()
    rec["build_s"] = time.perf_counter() - t0
    del X
    cap = ix.hnsw_out_cap()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    rec.update({"rows": N, "dim": D, "storage": "f16", "metric": "cosine", "ef_search": ef, "levels": LEVELS, "none_width": cap,
                "hnsw": []})
    print(f"{'batch':>5} | {'k=10 ms':>9} {'None ms':>9} {'ratio':>6} {'mean None count':>15}")
    for B in (1, 64, 1024):
        reps = {1: 40, 64: 15, 1024: 5}[B]
        q = Q[:B].contiguous()
        row = {"batch": B}
        for name, k, kw in (("top10", 10, {}), ("none", cap, {"all_candidates": True})):
            ids = torch.zeros((B, k), dtype=torch.int32, device=dev)
            scores = torch.zeros((B, k), dtype=torch.float32, device=dev)
            counts = torch.zeros(B, dtype=torch.int32, device=dev)

            def call():
                ix.batch_search_device(q.data_ptr(), B, k, ids.data_ptr(), scores.data_ptr(), counts.data_ptr(), None, stream.cuda_stream,
                                       mode=cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64, **kw)

            call()
            stream.synchronize()
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                call()
                e1.record(stream)
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            row[name + "_ms"] = float(np.median(ts))
            row[name + "_mean_count"] = float(counts.float().mean())
        print(f"{B:>5} | {row['top10_ms']:>9.3f} {row['none_ms']:>9.3f} {row['none_ms'] / row['top10_ms']:>6.2f} "
              f"{row['none_mean_count']:>15.1f}")
        rec["hnsw"].append(row)
    ix.close()


def sharded_part(rec):
    import cosdata_b200 as cdb
    from cosdata_b200.sharding import ShardGroup, merge_packed, pack_keys
    from oracle import pymeta
    from tests import mdgraph

    B, k, D, n = 1024, 10, 128, 3000
    shards, vecs0, mg0 = [], None, None
    for s in range(2):
        vecs, mg = mdgraph.build(n=n, dim=D, md_dims=6, levels=5, nb=16, nb0=32, storage_type=int(cdb.StorageType.HalfPrecisionFP),
                                 metric=0, seed=51 + s)
        fg = mg.fg
        ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=vecs.shape[0], keep_raw_f32=True,
                            id_base=s << 24)
        ix.append(vecs)
        ix.set_graph(fg.num_levels, fg.neighbors_count, fg.level0_neighbors_count, fg.entry, fg.n, fg.node_row, fg.adj, fg.child)
        node_id = [np.where(a < pymeta.PSEUDO_ROOT_ID, a + (s << 24), a).astype(np.uint32) for a in mg.node_id]
        ix.set_graph_metadata(mg.md_bits, mg.md_mags, node_id, mg.node_md, mg.pseudo_entry)
        shards.append(ix)
        if s == 0:
            vecs0, mg0 = vecs, mg
    g = ShardGroup.local([0, 0])
    for s, ix in enumerate(shards):
        g.attach(s, ix)
    q, filters = mdgraph.make_queries(vecs0, mg0, B, seed=9)
    filters = [None if i % 4 == 0 else f[:1] for i, f in enumerate(filters)]

    def group():
        return g.search_filtered(q, filters, k, ef_search=64)

    def per_shard():
        per = [ix.batch_search_filtered(q, filters, k, ef_search=64) for ix in shards]
        ids, scores, counts = merge_packed(np.stack([pack_keys(r[0], r[1]) for r in per]), k)
        return ids, scores, counts, np.bitwise_or.reduce(np.stack([r[3] for r in per]), axis=0)

    out = {}
    for name, fn in (("group", group), ("per_shard_numpy", per_shard)):
        fn()
        ts = []
        for _ in range(7):
            t0 = time.perf_counter()
            res = fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        out[name] = (float(np.median(ts)), res)
    same = all(np.array_equal(np.asarray(a).view(np.uint32) if np.asarray(a).dtype == np.float32 else a,
                              np.asarray(b).view(np.uint32) if np.asarray(b).dtype == np.float32 else b)
               for a, b in zip(out["group"][1], out["per_shard_numpy"][1]))
    rec["sharded_filtered"] = {"shards": 2, "embeddings_per_shard": n, "dim": D, "batch": B, "k": k, "group_ms": out["group"][0],
                               "per_shard_numpy_ms": out["per_shard_numpy"][0], "same_results": bool(same)}
    print(f"filtered sharded, 2 loopback shards, batch {B}: group {out['group'][0]:.2f} ms, per-shard + numpy merge "
          f"{out['per_shard_numpy'][0]:.2f} ms, results {'equal' if same else 'DIFFER'}")
    g.close()
    for ix in shards:
        ix.close()
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    rec = {"card": card()}
    hnsw_part(args, rec)
    same = sharded_part(rec)
    print(json.dumps(rec))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
