"""Sharded sparse search with top_k None (cdb_sparse_search_batch_all_sharded) against what a caller had to do without it:
every shard's own cdb_sparse_search_batch_all, then a numpy merge of the shards' sorted lists by the library's ordering
rule (key = order_key(score) << 32 | ~id, descending).  The corpus is the 1M-row corpus of tools/bench_sparse_all.py,
split into --shards contiguous shards: a loopback group on one card, or one card per shard when the host has that many.
Per batch size and re-rank setting: median ms per call (min, max) after one warm-up, both paths ending with every result
in numpy.  Checks a sample of queries of the two paths for equal offsets, ids and score bits.  Prints the card and its
power limit, read in the same run, and one JSON line.

    python tools/bench_sharded_sparse_all.py [--rows 1000000] [--shards 2] [--batches 1,64] [--steps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosdata_b200 as cdb  # noqa: E402
from cosdata_b200.sharding import ShardGroup, pack_keys, shard_range  # noqa: E402
from tests.sparse_data import slice_csr, zipf_csr  # noqa: E402

CHUNK = 500_000     # rows generated per call, as tools/bench_sparse_all.py


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def shim(shards, q, opts):
    """per-shard batch_search_all, then a host merge of each query's sorted runs"""
    parts = [s.batch_search_all(q, opts) for s in shards]
    nq = len(parts[0][0]) - 1
    counts = sum(np.diff(p[0].astype(np.int64)) for p in parts)
    off = np.zeros(nq + 1, np.uint64)
    off[1:] = np.cumsum(counts)
    ids = np.empty(int(off[-1]), np.uint32)
    scores = np.empty(int(off[-1]), np.float32)
    for i in range(nq):
        seg_ids = np.concatenate([p[1][int(p[0][i]):int(p[0][i + 1])] for p in parts])
        seg_sc = np.concatenate([p[2][int(p[0][i]):int(p[0][i + 1])] for p in parts])
        order = np.argsort(pack_keys(seg_ids, seg_sc), kind="stable")[::-1]
        b = int(off[i])
        ids[b:b + len(order)] = seg_ids[order]
        scores[b:b + len(order)] = seg_sc[order]
    return off, ids, scores


def timed(call, steps):
    out = call()                                   # warm-up
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = call()                               # each call ends with its results in host memory
        times.append((time.perf_counter() - t0) * 1e3)
    return out, float(np.median(times)), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--sample", default="0,1,63")
    a = ap.parse_args()
    assert cdb.device_count() > 0, "needs a CUDA device"
    name = card()
    n, ub = a.rows, 3.0
    corpus = [zipf_csr(1000 + i, min(CHUNK, n - r0)) for i, r0 in enumerate(range(0, n, CHUNK))]
    devs = list(range(a.shards)) if cdb.device_count() >= a.shards else [0] * a.shards
    g = ShardGroup.local(devs)
    shards = []
    for r in range(a.shards):
        row0, rows = shard_range(n, a.shards, r)
        pieces = []
        for i, c in enumerate(corpus):                 # the pieces of the generated chunks that fall in [row0, row0 + rows)
            c0 = i * CHUNK
            lo, hi = max(row0, c0), min(row0 + rows, c0 + len(c[0]) - 1)
            if lo < hi:
                pieces.append(slice_csr(c, lo - c0, hi - c0))
        ix = cdb.SparseIndex(quantization_bits=4, values_upper_bound=ub, capacity_rows=rows,
                             capacity_pairs=sum(len(p[1]) for p in pieces), id_base=row0, device=devs[r])
        for p in pieces:
            ix.append(p)
        g.attach_sparse(r, ix)
        shards.append(ix)
    queries = zipf_csr(7, 1024, mean_pairs=40)
    sample = [int(x) for x in a.sample.split(",")]
    res = dict(card=name, rows=n, shards=a.shards, devices=devs, steps=a.steps)
    for b in (int(x) for x in a.batches.split(",")):
        q = slice_csr(queries, 0, b)
        for rerank in (False, True):
            opts = cdb.SparseSearchOptions(None, 0.0, rerank)
            got, ms, lo, hi = timed(lambda: g.search_sparse_all(q, opts), a.steps)
            want, s_ms, s_lo, s_hi = timed(lambda: shim(shards, q, opts), a.steps)
            ok = True
            for i in (s for s in sample if s < b):
                bg, eg, bw, ew = int(got[0][i]), int(got[0][i + 1]), int(want[0][i]), int(want[0][i + 1])
                ok &= bg == bw and eg == ew and np.array_equal(got[1][bg:eg], want[1][bw:ew]) and \
                    np.array_equal(got[2][bg:eg].view(np.uint32), want[2][bw:ew].view(np.uint32))
            tag = f"b{b}_{'rerank' if rerank else 'plain'}"
            res[tag] = dict(group_ms=round(ms, 2), group_min_max=[round(lo, 2), round(hi, 2)], shim_ms=round(s_ms, 2),
                            shim_min_max=[round(s_lo, 2), round(s_hi, 2)], results=int(got[0][-1]), parity_sample=bool(ok))
            print(tag, json.dumps(res[tag]), flush=True)
    g.close()
    for s in shards:
        s.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
