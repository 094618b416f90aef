"""Cost of making a loaded replica graph writable (cdb_index_set_graph_slot_scores) and of writing to it, against a graph built
on the handle.

  (a) attach: a synthetic graph with --attach-nodes level-0 nodes (comma-separated sizes; 64 level-0 and 32 upper neighbours,
      every slot filled, upper levels a quarter of the one below) is uploaded with its metadata, then the stored slot values
      and tags are attached.  Reported per size: the call's host-clock time, and from a torch.profiler trace of a second
      attach the summed host-to-device copies and the summed attach kernels (hnsw_attach_*).
  (b) writes: a replica graph of 0.9 N embeddings (bench_insert_replicas' population and c3 rows, f16, cosine, reference
      defaults) is built on one handle; a second handle gets the same graph through set_graph + set_graph_metadata + its
      slot similarities (what a cold start from the index files holds).  Both then insert the other 0.1 N embeddings and
      delete 1 % of the rows, max_batch 4096.  Reported: seconds and nodes (rows) per second of each.

Times are host clocks around calls that end in a device synchronise.  Prints one JSON line with the card name and power limit.

    python tools/bench_loaded_graph.py [--attach-nodes 1000000,10000000] [--rows 200000] [--dim 768]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_insert_replicas import card, population   # noqa: E402

EMPTY = 0xFFFFFFFF


def synthetic_graph(n0, rng):
    """level arrays of a graph with n0 level-0 nodes (node i = row i), every slot filled with a random other node"""
    counts = [n0]
    while counts[-1] // 4 >= 64 and len(counts) < 10:
        counts.append(counts[-1] // 4)
    nbs = [64] + [32] * (len(counts) - 1)
    node_row, adj, child = [], [], []
    for lv, (c, nb) in enumerate(zip(counts, nbs)):
        node_row.append(np.arange(c, dtype=np.uint32))
        a = rng.integers(0, c - 1, (c, nb), dtype=np.uint32)
        a += (a >= np.arange(c, dtype=np.uint32)[:, None])   # no self links
        adj.append(a.ravel())
        child.append(np.arange(c, dtype=np.uint32))           # node i of level L is node i of level L - 1
    return counts, nbs, node_row, adj, child


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--attach-nodes", default="1000000,10000000")
    ap.add_argument("--rows", type=int, default=200_000)
    ap.add_argument("--dim", type=int, default=768)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ST, MK = cdb.StorageType.HalfPrecisionFP, cdb.DistanceMetricKind.Cosine
    rec = {"card": card(), "attach": {}, "writes": {}}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    # ---- (a) attach
    rng = np.random.default_rng(1)
    for n0 in [int(x) for x in args.attach_nodes.split(",") if x]:
        counts, nbs, node_row, adj, child = synthetic_graph(n0, rng)
        L = len(counts) - 1
        ix = cdb.DenseIndex(dim=16, storage_type=cdb.StorageType.UnsignedByte, metric=MK, capacity=n0, keep_raw_f32=False)
        for a in range(0, n0, 1 << 20):
            ix.append(rng.uniform(-0.9, 0.9, (min(1 << 20, n0 - a), 16)).astype(np.float32))
        ix.set_graph(L, 32, 64, 0, 0, node_row, adj, child)
        ids = [np.arange(c, dtype=np.uint32) for c in counts]
        mds = [np.zeros(c, np.uint32) for c in counts]
        md_bits, md_mags = np.zeros((1, 6), np.int32), np.zeros(1, np.float32)
        scores = [rng.uniform(-1, 1, a.size).astype(np.float32) for a in adj]
        tags = [np.zeros(a.size, np.uint8) for a in adj]
        ix.set_graph_metadata(md_bits, md_mags, ids, mds, 0)
        t, _ = timed(lambda: ix.set_graph_slot_scores(scores, tags))
        ix.set_graph_metadata(md_bits, md_mags, ids, mds, 0)   # drops the state: attach again under the profiler
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ix.set_graph_slot_scores(scores, tags)
            torch.cuda.synchronize()
        h2d = kern = 0.0
        for e in prof.events():
            dur = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "HtoD" in e.name:
                h2d += dur
            elif e.name.startswith("hnsw_attach") or "hnsw_attach" in e.name:
                kern += dur
        slots = int(sum(a.size for a in adj))
        rec["attach"][str(n0)] = {"levels": L + 1, "slots": slots, "call_s": t, "h2d_copies_ms": h2d / 1000.0,
                                  "attach_kernels_ms": kern / 1000.0, "h2d_bytes": slots * 5}
        ix.close()
        del scores, tags, adj
    # ---- (b) inserts and deletes: built on the handle vs loaded
    N, D, LEVELS = args.rows, args.dim, 9
    n0 = N - N // 10
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    centres = torch.randn((4096, D), generator=g, device=dev)
    X = ((centres[torch.randint(0, 4096, (N,), generator=g, device=dev)] + 0.35 * torch.randn((N, D), generator=g, device=dev))
         / (4.5 * 1.06)).clamp_(-0.999, 0.999).contiguous()
    pop = population(N, LEVELS)
    body, pseudo = pop["body"], pop["pseudo"]
    emb = body["row"].astype(np.int64)

    def nodes(lo, hi, shift):
        a, b = np.searchsorted(emb, lo), np.searchsorted(emb, hi)
        part = {c: v[a:b] for c, v in body.items()}
        part["row"] = (part["row"] + shift).astype(np.uint32)
        return part

    built = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 2, keep_raw_f32=True)
    built.append_device(X[:n0].data_ptr(), n0)
    part = nodes(0, n0, 0)
    lst = {c: np.concatenate([pseudo[c], part[c]]) for c in part}
    built.build_graph_replicas(lst["row"], lst["node_id"], lst["base_id"], lst["md_row"], lst["max_level"], pop["md_bits"],
                               pop["md_mags"], 0, 1, LEVELS, 32, 64, 128, 64, 4096, 1)
    gr = built.read_graph()
    gids, gmds = built.read_graph_metadata()
    # the same rows (the roots' codes are the build's; their raw rows never reach a result) and the same graph
    roots = np.zeros((2, D), np.float32)
    loaded = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 2, keep_raw_f32=True)
    c_all, m_all = built.read_codes(0, n0 + 2)
    loaded.append_codes(c_all, m_all)
    loaded.set_raw(0, np.concatenate([X[:n0].cpu().numpy(), roots]))
    loaded.set_graph(gr["num_levels"], 32, 64, gr["entry"], gr["root_row"], gr["node_row"], gr["adj"], gr["child"])
    loaded.set_graph_metadata(pop["md_bits"], pop["md_mags"], gids, gmds, 1)
    t_attach, _ = timed(lambda: loaded.set_graph_slot_scores(built.read_replica_slot_scores()))
    rec["writes"]["graph_nodes"] = int(gr["node_row"][0].size)
    rec["writes"]["attach_s"] = t_attach
    new = nodes(n0, N, 2)
    dead = np.random.default_rng(2).choice(n0, N // 100, replace=False).astype(np.uint32)
    for name, ix in (("built", built), ("loaded", loaded)):
        ix.append_device(X[n0:].data_ptr(), N - n0)
        ti, f = timed(lambda: ix.insert_graph_replicas(new["row"], new["node_id"], new["base_id"], new["md_row"], new["max_level"],
                                                       ef_construction=128, shortlist_size=64, max_batch=4096))
        td, s = timed(lambda: ix.delete_rows_replicas(dead, 64, 4096))
        rec["writes"][name] = {"insert_nodes": int(f.size), "insert_s": ti, "insert_nodes_per_s": f.size / ti, "insert_failed": int(f.sum()),
                               "delete_rows": int(dead.size), "delete_s": td, "delete_rows_per_s": dead.size / td,
                               "delete_status2": int((s == 2).sum())}
        ix.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
