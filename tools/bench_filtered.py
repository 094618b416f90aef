"""Filtered HNSW search on a replica graph (a collection with a metadata schema): the device entry point and the host one.

The graph: N embeddings (default 1M) of bench.py's clustered c3 rows, 768-dim f16 storage with raw f32 rows kept, cosine,
the node population of tools/bench_insert_replicas.py (7 pseudo replicas; per embedding a base replica and, for two thirds
of the embeddings, one or two metadata replicas over 7 patterns of 6 binary dimensions), built on the GPU with
build_graph_replicas (9 levels, 32/64 neighbours, ef_construction 128).  Workloads: ef 128, k 10, batches of 1, 64 and 1024
queries, each unfiltered, with one filter and with three filters per query.  Per workload the device form runs on one stream
(ms per call from CUDA events, median after warm-up), the host form is timed with a host clock around its synchronising
call, and the ids, counts, score bits and error flags of every timed device batch are compared with the first one's and the
host form's.  Prints a table, the parity line and one JSON line with the card name and power limit of the same run.

    python tools/bench_filtered.py [--rows 1000000] [--dim 768]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_insert_replicas import N_PATTERNS, card, population  # noqa: E402

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    args = ap.parse_args()
    import torch
    import cosdata_b200 as cdb

    N, D, k, ef, LEVELS = args.rows, args.dim, 10, 128, 9
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
    Q = draw(1024)
    pop = population(N, LEVELS)
    body, pseudo = pop["body"], pop["pseudo"]
    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.HalfPrecisionFP, metric=cdb.DistanceMetricKind.Cosine, capacity=N + 2,
                        keep_raw_f32=True)
    ix.append_device(X.data_ptr(), N)
    lst = {c: np.concatenate([pseudo[c], body[c]]) for c in body}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    failed = ix.build_graph_replicas(lst["row"], lst["node_id"], lst["base_id"], lst["md_row"], lst["max_level"], pop["md_bits"],
                                     pop["md_mags"], 0, 1, LEVELS, 32, 64, 128, 64, 4096, 1)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    del X
    pats = pop["md_bits"][2:].astype(np.int8)
    stream = torch.cuda.Stream()
    rec = {"card": card(), "embeddings": N, "graph_nodes": int(lst["row"].size + 2), "dim": D, "storage": "f16", "metric": "cosine",
           "ef_search": ef, "k": k, "build_s": build_s, "build_failed": int(failed.sum()), "workloads": []}
    parity_batches, parity_ok = 0, True
    print(f"{'batch':>5} {'filters':>7} | {'device ms':>9} {'host ms':>9}")
    for B in (1, 64, 1024):
        reps = {1: 40, 64: 15, 1024: 5}[B]
        for nf in (0, 1, 3):
            q = Q[:B].contiguous()
            filters = [None] * B if nf == 0 else [[pats[(i + j) % N_PATTERNS] for j in range(nf)] for i in range(B)]
            offs, dims, has = ix.pack_filters(filters)
            d_offs = torch.from_numpy(offs.view(np.int32)).to(dev)
            d_dims = torch.from_numpy(dims if dims.size else np.zeros((1, ix.md_dims), np.int8)).to(dev)
            d_has = torch.from_numpy(has).to(dev) if nf else None
            ids = torch.zeros((B, k), dtype=torch.int32, device=dev)
            scores = torch.zeros((B, k), dtype=torch.float32, device=dev)
            counts = torch.zeros(B, dtype=torch.int32, device=dev)
            err = torch.zeros(B, dtype=torch.uint8, device=dev)
            stream.wait_stream(torch.cuda.current_stream())

            def device_call():
                ix.batch_search_filtered_device(q.data_ptr(), B, k, d_offs.data_ptr(), d_dims.data_ptr(), dims.shape[0],
                                                None if d_has is None else d_has.data_ptr(), ids.data_ptr(), scores.data_ptr(),
                                                counts.data_ptr(), err.data_ptr(), stream.cuda_stream, ef_search=ef, shortlist_size=64)

            def timed_device():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                device_call()
                e1.record(stream)
                e1.synchronize()
                out = (ids.cpu().numpy().copy(), scores.cpu().numpy().view(np.uint32).copy(), counts.cpu().numpy().copy(),
                       err.cpu().numpy().copy())
                return e0.elapsed_time(e1), out

            _, ra = timed_device()   # warm-up
            tw = []
            for _ in range(reps):
                a, rb = timed_device()
                tw.append(a)
                parity_batches += 1
                parity_ok &= all(np.array_equal(x, y) for x, y in zip(ra, rb))
            qh = q.cpu().numpy()
            p = ix.params(k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64)
            hids, hsc = np.zeros((B, k), np.uint32), np.zeros((B, k), np.float32)
            hcnt, herr = np.zeros(B, np.uint32), np.zeros(B, np.uint8)
            hdims = dims if dims.size else np.zeros((1, ix.md_dims), np.int8)
            ptr = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731

            def host_call():
                return ix._lib.cdb_search_batch_filtered(ix._h, ptr(qh), B, C.byref(p), ptr(offs), ptr(hdims), ptr(has) if nf else None,
                                                         ptr(hids), ptr(hsc), ptr(hcnt), ptr(herr))
            assert host_call() == 0
            th = []
            for _ in range(reps):
                t0 = time.perf_counter()
                host_call()
                th.append((time.perf_counter() - t0) * 1e3)
            parity_ok &= np.array_equal(hids, ra[0].view(np.uint32)) and np.array_equal(hsc.view(np.uint32), ra[1])
            parity_ok &= np.array_equal(hcnt, ra[2].view(np.uint32)) and np.array_equal(herr, ra[3])
            w, h = float(np.median(tw)), float(np.median(th))
            print(f"{B:>5} {nf:>7} | {w:>9.3f} {h:>9.3f}")
            rec["workloads"].append({"batch": B, "filters_per_query": nf, "warp_ms": w, "host_form_ms": h, "warp_qps": B / w * 1e3,
                                     "mean_count": float(counts.float().mean())})
    print(f"parity: {'ok' if parity_ok else 'MISMATCH'} (ids, counts, score bits, error flags of {parity_batches} timed device "
          f"batches equal to the first one's; host form = device form)")
    rec["parity"] = bool(parity_ok)
    print(json.dumps(rec))
    ix.close()
    return 0 if parity_ok else 1


if __name__ == "__main__":
    sys.exit(main())
