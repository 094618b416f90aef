"""Cost of deleting embeddings from a replica graph (a collection with a metadata schema) on the GPU
(cdb_index_delete_rows_replicas), and the graph's recall afterwards.

On the population of tools/bench_insert_replicas.py (clustered f16 rows from bench.py's c3 generator, cosine, the reference
defaults: 9 levels, 32/64 neighbours, ef_construction 128; 7 pseudo replicas, per embedding a base replica and for two
thirds of the embeddings one or two metadata replicas), after a one-shot replica build of N embeddings this measures
  (a) `--singles` deletes of one embedding per call (per-call times);
  (b) one call deleting 10k embeddings;
  (c) one call deleting 100k embeddings;
then recall@10 at ef_search 128 for 1024 unfiltered and 1024 filtered queries (one pattern each) against the exact top-10
over the live embeddings, for the repaired graph and for a fresh replica build over the live embeddings only.  Times are
host clocks around calls that end in a device synchronise.  Prints one JSON line with the card name and power limit.

    python tools/bench_delete_replicas.py [--rows 1000000] [--dim 768] [--singles 1000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_insert_replicas import N_PATTERNS, REPLICAS, card, population  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--singles", type=int, default=1000)
    ap.add_argument("--queries", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb

    N, D, B, k, LEVELS = args.rows, args.dim, args.queries, 10, 9
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
    Q = draw(B)
    queries = Q.cpu().numpy()
    pop = population(N, LEVELS)
    body, pseudo = pop["body"], pop["pseudo"]
    lst = {c: np.concatenate([pseudo[c], body[c]]) for c in body}
    ST, MK = cdb.StorageType.HalfPrecisionFP, cdb.DistanceMetricKind.Cosine
    rng = np.random.default_rng(5)
    order = rng.permutation(N)
    n1, n2, n3 = args.singles, 10_000, 100_000
    dead = order[: n1 + n2 + n3]

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def index_built(keep):
        ix = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 2, keep_raw_f32=True)
        ix.append_device(X.data_ptr(), N)
        sel = keep[np.minimum(lst["row"], N - 1)] | (lst["row"] == 0xFFFFFFFF)
        t, f = timed(lambda: ix.build_graph_replicas(lst["row"][sel], lst["node_id"][sel], lst["base_id"][sel], lst["md_row"][sel],
                                                     lst["max_level"][sel], pop["md_bits"], pop["md_mags"], 0, 1, LEVELS, 32, 64, 128,
                                                     64, 4096, 1))
        return ix, t, int(f.sum())

    # exact top-10 over the live embeddings that qualify: unfiltered (all) and filtered (query q asks for pattern q % 7)
    live = np.ones(N, bool)
    live[dead] = False
    qpat = np.arange(B) % N_PATTERNS
    filters = [[pop["md_bits"][2 + int(p)].astype(np.int8)] for p in qpat]
    carries = torch.from_numpy(np.stack([(pop["patterns_of"] == p).any(1) & live for p in range(N_PATTERNS)])).to(dev)
    live_d = torch.from_numpy(live).to(dev)
    Xn = X / X.norm(dim=1, keepdim=True)
    Qn = Q / Q.norm(dim=1, keepdim=True)
    gt_all, gt_f = [], []
    for a in range(0, B, 128):
        s = Qn[a:a + 128] @ Xn.T
        s.masked_fill_(~live_d[None, :], float("-inf"))
        gt_all.append(s.topk(k, dim=1).indices.cpu())
        s.masked_fill_(~carries[torch.from_numpy(qpat[a:a + 128]).to(dev)], float("-inf"))
        gt_f.append(s.topk(k, dim=1).indices.cpu())
        del s
    gt_all, gt_f = torch.cat(gt_all).numpy(), torch.cat(gt_f).numpy()
    del Xn, carries

    def recall(ix):
        out = {}
        for name, flt, gt in (("unfiltered", [None] * B, gt_all), ("filtered", filters, gt_f)):
            ids, _, counts, _ = ix.batch_search_filtered(queries, flt, k, ef_search=128, shortlist_size=64)
            rows = ids // REPLICAS
            out[name] = sum(len(set(rows[i, : counts[i]].tolist()) & set(gt[i].tolist())) for i in range(B)) / (B * k)
            out[name + "_deleted_returned"] = int(sum((~live[rows[i, : counts[i]]]).sum() for i in range(B)))
        return out

    rec = {"card": card(), "embeddings": N, "graph_nodes": int(lst["row"].size + 2), "dim": D, "storage": "f16", "metric": "cosine",
           "params": {"num_levels": LEVELS, "neighbors": [32, 64], "ef_construction": 128}, "times_s": {}, "status2": {},
           "recall_at_10": {}}
    ix, t, f = index_built(np.ones(N, bool))
    rec["times_s"]["build_all"] = t
    per, s2 = [], 0
    for r in order[:n1]:   # (a)
        t, s = timed(lambda: ix.delete_rows_replicas([int(r)]))
        per.append(t)
        s2 += int((s == 2).sum())
    rec["times_s"]["a_single_mean"] = float(np.mean(per))
    rec["times_s"]["a_single_median"] = float(np.median(per))
    rec["times_s"]["a_singles_total"] = float(np.sum(per))
    rec["status2"]["a"] = s2
    t, s = timed(lambda: ix.delete_rows_replicas(order[n1:n1 + n2]))   # (b)
    rec["times_s"]["b_10k_call"] = t
    rec["status2"]["b"] = int((s == 2).sum())
    t, s = timed(lambda: ix.delete_rows_replicas(order[n1 + n2:n1 + n2 + n3]))   # (c)
    rec["times_s"]["c_100k_call"] = t
    rec["status2"]["c"] = int((s == 2).sum())
    rec["recall_at_10"]["repaired"] = recall(ix)
    ix.close()
    fx, t, f = index_built(live)
    rec["times_s"]["fresh_build_live"] = t
    rec["recall_at_10"]["fresh_build_live"] = recall(fx)
    fx.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
