"""Cost of growing a replica graph (a collection with a metadata schema) on the GPU (cdb_index_insert_graph_replicas) against
building it in one go (cdb_index_build_graph_replicas).

On clustered rows from bench.py's c3 generator (f16 storage, cosine, the reference defaults: 9 levels, 32/64 neighbours,
ef_construction 128), with the node population of tests/mdgraph.replica_population (7 pseudo replicas created with the
collection; per embedding a base replica, and for two thirds of the embeddings one or two metadata replicas over 7 patterns
of 6 binary dimensions), this measures
  (a) a one-shot replica build of N embeddings;
  (b) a build of 0.9 N embeddings + one insert of the other 0.1 N;
  (c) a build of 0.9 N embeddings + `--calls` inserts of 0.1 N / calls embeddings each (per-call times);
and recall@10 at ef_search 128 of (a), (b) and (c) for 1024 unfiltered queries (against the exact top-10 over all
embeddings) and 1024 filtered ones (one pattern each, against the exact top-10 over the embeddings that carry it).  Times are
host clocks around calls that end in a device synchronise.  Prints one JSON line with the card name and power limit.

    python tools/bench_insert_replicas.py [--rows 1000000] [--dim 768] [--calls 100]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EMPTY = 0xFFFFFFFF
PSEUDO_ROOT_ID = 0xFFFFFFFF - 257
REPLICAS = 4            # replica ids of embedding i: i * REPLICAS + j
N_PATTERNS, MD_DIMS = 7, 6


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def population(n, levels, seed=3):
    """the replica list of n embeddings in insertion order (as tests/mdgraph.replica_population builds it, vectorised):
    -> dict(row, node_id, base_id, md_row, max_level) with rows = embedding index (pseudo replicas: EMPTY), md_bits, md_mags,
    patterns_of [n, 2] (-1 = none)"""
    from cosdata_b200.api import level_probs, max_insert_level, pseudo_level_probs
    rng = np.random.default_rng(seed)
    patterns = np.array([[((p + 1) >> b) & 1 for b in range(MD_DIMS)] for p in range(N_PATTERNS)], np.int32)
    md_bits = np.concatenate([np.zeros((1, MD_DIMS), np.int32), np.ones((1, MD_DIMS), np.int32), patterns])
    md_mags = np.sqrt((md_bits.astype(np.float64) ** 2).sum(1)).astype(np.float32)   # Metadata.mag of 0/1 dimensions
    md_mags[0] = 0.0
    i = np.arange(n)
    p = rng.integers(0, N_PATTERNS, (n, 2))
    nf = np.where(i % 3 == 0, 0, 1 + i % 2)
    nf = np.where((nf == 2) & (p[:, 0] == p[:, 1]), 1, nf)
    p = np.sort(p, axis=1)
    patterns_of = np.where(np.arange(2)[None, :] < nf[:, None], p, -1)
    per = 1 + nf
    emb = np.repeat(i, per)
    j = np.arange(emb.size) - np.repeat(np.cumsum(per) - per, per)       # replica index within the embedding
    md = np.where(j == 0, 0, 2 + patterns_of[emb, np.maximum(j - 1, 0)])
    th = np.array([1.0 - 4.0 ** (-m) for m in range(1, levels + 1)])
    lv = np.searchsorted(th, rng.random(emb.size).astype(np.float32), side="right")
    plp = pseudo_level_probs(levels, N_PATTERNS)
    ps = dict(row=np.full(N_PATTERNS, EMPTY), node_id=PSEUDO_ROOT_ID + 1 + np.arange(N_PATTERNS),
              base_id=np.full(N_PATTERNS, PSEUDO_ROOT_ID), md_row=2 + np.arange(N_PATTERNS),
              max_level=np.array([max_insert_level(float(np.float32(x)), plp) for x in rng.random(N_PATTERNS)]))
    body = dict(row=emb, node_id=emb * REPLICAS + j, base_id=emb * REPLICAS, md_row=md, max_level=lv)
    out = {c: (ps[c], body[c]) for c in ps}
    return dict(pseudo={c: np.asarray(v[0], np.uint8 if c == "max_level" else np.uint32) for c, v in out.items()},
                body={c: np.asarray(v[1], np.uint8 if c == "max_level" else np.uint32) for c, v in out.items()},
                md_bits=md_bits, md_mags=md_mags, patterns_of=patterns_of)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--queries", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb

    N, D, B, k, LEVELS = args.rows, args.dim, args.queries, 10, 9
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
    Q = draw(B)
    queries = Q.cpu().numpy()
    pop = population(N, LEVELS)
    body, pseudo = pop["body"], pop["pseudo"]
    emb = body["row"].astype(np.int64)
    # exact top-10 over the embeddings that qualify: unfiltered (all) and filtered (query q asks for pattern q % 7)
    qpat = np.arange(B) % N_PATTERNS
    filters = [[pop["md_bits"][2 + int(p)].astype(np.int8)] for p in qpat]
    carries = torch.from_numpy(np.stack([(pop["patterns_of"] == p).any(1) for p in range(N_PATTERNS)])).to(dev)   # [7, N]
    Xn = X / X.norm(dim=1, keepdim=True)
    Qn = Q / Q.norm(dim=1, keepdim=True)
    gt_all, gt_f = [], []
    for a in range(0, B, 128):
        s = Qn[a:a + 128] @ Xn.T
        gt_all.append(s.topk(k, dim=1).indices.cpu())
        s.masked_fill_(~carries[torch.from_numpy(qpat[a:a + 128]).to(dev)], float("-inf"))
        gt_f.append(s.topk(k, dim=1).indices.cpu())
        del s
    gt_all, gt_f = torch.cat(gt_all).numpy(), torch.cat(gt_f).numpy()
    del Xn, carries
    torch.cuda.synchronize()
    ST, MK = cdb.StorageType.HalfPrecisionFP, cdb.DistanceMetricKind.Cosine

    def index(rows):
        ix = cdb.DenseIndex(dim=D, storage_type=ST, metric=MK, capacity=N + 2, keep_raw_f32=True)
        ix.append_device(X[:rows].data_ptr(), rows)
        return ix

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def recall(ix):
        out = {}
        for name, flt, gt in (("unfiltered", [None] * B, gt_all), ("filtered", filters, gt_f)):
            ids, _, counts, _ = ix.batch_search_filtered(queries, flt, k, ef_search=128, shortlist_size=64)
            hits = sum(len(set((ids[i, : counts[i]] // REPLICAS).tolist()) & set(gt[i].tolist())) for i in range(B))
            out[name] = hits / (B * k)
        return out

    def nodes(lo, hi, shift):   # the list entries of embeddings [lo, hi), rows shifted behind the two roots
        a, b = np.searchsorted(emb, lo), np.searchsorted(emb, hi)
        part = {c: v[a:b] for c, v in body.items()}
        part["row"] = (part["row"] + shift).astype(np.uint32)
        return part

    def build(ix, n_emb):
        part = nodes(0, n_emb, 0)
        lst = {c: np.concatenate([pseudo[c], part[c]]) for c in part}
        return timed(lambda: ix.build_graph_replicas(lst["row"], lst["node_id"], lst["base_id"], lst["md_row"], lst["max_level"],
                                                     pop["md_bits"], pop["md_mags"], 0, 1, LEVELS, 32, 64, 128, 64, 4096, 1))

    def insert(ix, lo, hi):
        ix.append_device(X[lo:hi].data_ptr(), hi - lo)
        part = nodes(lo, hi, 2)
        return timed(lambda: ix.insert_graph_replicas(part["row"], part["node_id"], part["base_id"], part["md_row"], part["max_level"],
                                                      ef_construction=128, shortlist_size=64, max_batch=4096))

    rec = {"card": card(), "embeddings": N, "graph_nodes": int(emb.size + N_PATTERNS + 2), "dim": D, "storage": "f16",
           "metric": "cosine", "params": {"num_levels": LEVELS, "neighbors": [32, 64], "ef_construction": 128},
           "times_s": {}, "recall_at_10": {}, "failed": {}}
    # (a) one-shot build
    ix = index(N)
    t, f = build(ix, N)
    rec["times_s"]["a_build_all"] = t
    rec["failed"]["a"] = int(f.sum())
    rec["recall_at_10"]["a"] = recall(ix)
    ix.close()
    # (b) build 0.9 N + one insert of 0.1 N
    ix = index(n0)
    t, _ = build(ix, n0)
    rec["times_s"]["b_build_0.9"] = t
    t, f = insert(ix, n0, N)
    rec["times_s"]["b_insert_0.1"] = t
    rec["b_insert_nodes"] = int(f.size)
    rec["failed"]["b"] = int(f.sum())
    rec["recall_at_10"]["b"] = recall(ix)
    ix.close()
    # (c) build 0.9 N + `calls` inserts
    ix = index(n0)
    t, _ = build(ix, n0)
    rec["times_s"]["c_build_0.9"] = t
    per, failed = [], 0
    step = (N - n0) // args.calls
    for c in range(args.calls):
        a = n0 + c * step
        b = N if c == args.calls - 1 else a + step
        t, f = insert(ix, a, b)
        per.append(t)
        failed += int(f.sum())
    rec["times_s"]["c_inserts_total"] = float(np.sum(per))
    rec["times_s"]["c_insert_first10_mean"] = float(np.mean(per[:10]))
    rec["times_s"]["c_insert_last10_mean"] = float(np.mean(per[-10:]))
    rec["times_s"]["c_insert_max"] = float(np.max(per))
    rec["failed"]["c"] = failed
    rec["recall_at_10"]["c"] = recall(ix)
    ix.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
