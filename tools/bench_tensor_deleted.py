"""Cost of deleted rows on the brute-force tensor-core paths (CDB_SEARCH_TENSOR_WITH_DELETED, DESIGN.md section 5).

    python tools/bench_tensor_deleted.py --out DIR [--steps 5] [--warmup 2] [--exact-steps 2] [--c2-rows N] [--c4-rows N]

Shapes: C2 (brute-force cosine top-10 over 10M x 768 f32, B = 1024, the prefilter's f16 and s8 forms forced with
CDB_TS_S8) and a C4-like shard (quaternary codes, dot product, 5M x 1024, B = 4096, the u8 wgmma).  Deleted: 0.1 %, 1 % and
10 % of the rows drawn at random, and the pre-delete top-10 of every query.  For each case, on one index:
  (a) no deletes, (b) deleted rows without the flag (the exact scan), (c) deleted rows with the flag.
Per cell: ms per call (host clock around a synchronous search, after warm-up), the scan kernel's ms per chunk of <= 2048
queries (cdb_index_scan_ms_history) and candidates per query; (b) and (c) must return bit-identical ids, scores and counts.
The card's name and power limit are read in the same run.  Writes DIR/tensor_deleted.json and prints it as one line.
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

SEED_CORPUS = 0xC05DA7A + 2     # bench.py's C2 seeds
SEED_QUERY = 0xC05DA7A + 102
FORM = {"0": "f16", "1": "s8", None: "u8"}   # CDB_TS_S8 value -> the path it selects


def gpu_query(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    return [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else None


def timed(ix, q, k, mode, steps, warmup, form=None, **kw):
    """-> (cell dict, outputs) of `steps` synchronous searches after `warmup` ones"""
    if form is not None:
        os.environ["CDB_TS_S8"] = form
    st0 = ix.stats()
    for _ in range(warmup):
        ix.batch_search(q, k, mode, **kw)
    ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = ix.batch_search(q, k, mode, **kw)
        ms.append((time.perf_counter() - t0) * 1e3)
    st1 = ix.stats()
    os.environ.pop("CDB_TS_S8", None)
    chunks = (q.shape[0] + 2047) // 2048          # a call searches in chunks of <= 2048 queries
    calls = (steps + warmup) * chunks
    tensor = st1["tensor_searches"] - st0["tensor_searches"]
    cell = {"ms_call": float(np.median(ms)), "kernel_ms_per_chunk": float(np.median(ix.scan_ms_history(steps * chunks))),
            "tensor_path": bool(tensor == calls), "fallback_queries_last_chunk": st1["fallback_queries"] if tensor else None}
    if tensor:
        cell["cand_per_query_last_chunk"] = float(ix.last_candidate_counts(min(q.shape[0], 2048)).mean())
    if form is not None:
        cell["s8"] = st1["s8_searches"] - st0["s8_searches"] == calls
    return cell, out


def same(a, b):
    return all(np.array_equal(np.ascontiguousarray(x).view(np.uint32), np.ascontiguousarray(y).view(np.uint32))
               for x, y in zip(a, b))


def run_case(make, q, k, mode, forms, case, args):
    ix = make()
    n = ix.size
    rec = {"case": case}
    for f in forms:
        rec["a_" + FORM[f]], _ = timed(ix, q, k, mode, args.steps, args.warmup, f)
    if case == "top10":
        ids, _, _, _ = ix.batch_search(q, 10, mode)
        dead = np.unique(ids)
    else:
        dead = np.random.default_rng(11).choice(n, max(1, int(n * float(case))), replace=False)
    t0 = time.perf_counter()
    assert (ix.delete_rows(np.sort(dead).astype(np.uint32)) == 0).all()
    rec["deleted"] = int(dead.size)
    rec["delete_call_s"] = time.perf_counter() - t0
    rec["b_exact"], ob = timed(ix, q, k, mode, args.exact_steps, 1)
    assert not rec["b_exact"]["tensor_path"]
    rec["identical"] = True
    for f in forms:
        c, oc = timed(ix, q, k, mode, args.steps, args.warmup, f, tensor_with_deleted=True)
        assert c["tensor_path"], ("the tensor-core path did not run with the flag", case, f)
        rec["c_" + FORM[f]] = c
        rec["identical"] &= same(ob, oc)
    ix.close()
    assert rec["identical"], ("flag on / off outputs differ", rec)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--c2-rows", type=int, default=10_000_000)
    ap.add_argument("--c4-rows", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--exact-steps", type=int, default=2)
    ap.add_argument("--cases", default="0.001,0.01,0.1,top10")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = gpu_query("name,power.limit,clocks.max.sm")
    rec = {"gpu": info[0] if info else None, "power_limit_w": info[1] if info else None,
           "max_sm_clock_mhz": info[2] if info else None, "c2": [], "c4": []}
    cases = args.cases.split(",")

    q2 = cdb.synth_matrix(SEED_QUERY, 1024, 768)

    def make_c2():
        ix = cdb.DenseIndex(dim=768, capacity=args.c2_rows)
        ix.append_synthetic(SEED_CORPUS, args.c2_rows)
        return ix
    for case in cases:
        rec["c2"].append(run_case(make_c2, q2, 10, cdb.SearchMode.BRUTE_RAW, ["0", "1"], case, args))

    q4 = cdb.synth_matrix(SEED_QUERY + 4, 4096, 1024)

    def make_c4():
        ix = cdb.DenseIndex(dim=1024, storage_type=cdb.StorageType.SubByte2, metric=cdb.DistanceMetricKind.DotProduct,
                            capacity=args.c4_rows)
        ix.append_synthetic(SEED_CORPUS + 4, args.c4_rows)
        return ix
    for case in cases:
        rec["c4"].append(run_case(make_c4, q4, 10, cdb.SearchMode.BRUTE_CODES, [None], case, args))

    with open(os.path.join(args.out, "tensor_deleted.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
