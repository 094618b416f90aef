"""Kernel breakdown of the headline step (bench.py C2: brute-force cosine top-10, 10M x 768 f32, B = 1024).

    python tools/bench_rerank_overlap.py --out DIR [--rows N] [--rounds 3] [--steps 20] [--warmup 5] [--profile-steps 3]

1. --rounds rounds of --steps device searches, profiler off: ms per step (CUDA events), the s8 scan's ms
   (cdb_index_scan_ms_history), candidates per query, SM clock and board power during the round, and a bit-for-bit
   comparison of the rounds' outputs.
2. In a run of its own, torch.profiler (CUDA activity) over --profile-steps warm steps: device ms per step of every kernel.
The card's name and power limit are read in the same call.  Writes DIR/rerank_overlap.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED_CORPUS = 0xC05DA7A + 2     # bench.py
SEED_QUERY = 0xC05DA7A + 102


def gpu_query(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    return [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else None


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max()), "n": int(v.size)}


def kernel_breakdown(torch, step, steps):
    """device ms per step of every kernel name, from a torch.profiler trace of `steps` warm steps"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if str(getattr(ev, "device_type", "")) != "DeviceType.CUDA":
            continue
        us = getattr(ev, "device_time", None)
        if us is None:
            us = ev.cuda_time
        d = out.setdefault(ev.name.split("<")[0].split("(")[0], {"ms_per_step": 0.0, "launches_per_step": 0.0})
        d["ms_per_step"] += us / 1000.0 / steps
        d["launches_per_step"] += 1.0 / steps
    return dict(sorted(out.items(), key=lambda kv: -kv[1]["ms_per_step"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = gpu_query("name,power.limit,clocks.max.sm")
    rec = {"gpu": info[0] if info else None, "power_limit_w": info[1] if info else None,
           "max_sm_clock_mhz": info[2] if info else None, "rows": args.rows, "batch": args.batch}

    import torch
    import cosdata_b200 as cdb
    n, dim, B, k = args.rows, 768, args.batch, 10
    dev = torch.device("cuda", 0)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append_synthetic(SEED_CORPUS, n)
    d_q = torch.from_numpy(cdb.synth_matrix(SEED_QUERY, B, dim)).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    rec["sm_count"] = torch.cuda.get_device_properties(dev).multi_processor_count

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream)

    rounds, first = [], None
    for _ in range(args.rounds):
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        e1.record(stream)
        clk = gpu_query("clocks.sm,power.draw")
        torch.cuda.synchronize()
        cand = ix.last_candidate_counts(B)
        rounds.append({"ms_step": e0.elapsed_time(e1) / args.steps, "scan_ms": float(np.median(ix.scan_ms_history(args.steps))),
                       "cand_mean": float(cand.mean()), "sm_clock_mhz": float(clk[0]) if clk else None,
                       "power_w": float(clk[1]) if clk else None})
        o = (d_ids.cpu().numpy().copy(), d_scores.cpu().numpy().view(np.uint32).copy(), d_counts.cpu().numpy().copy())
        first = first or o
        assert all(np.array_equal(a, b) for a, b in zip(first, o)), "the step's output changed between rounds"
    st = ix.stats()
    rec["s8_searches"], rec["fallback_queries"] = st["s8_searches"], st["fallback_queries"]
    rec["summary"] = {key: stats([r[key] for r in rounds if r[key] is not None])
                      for key in ("ms_step", "scan_ms", "cand_mean", "sm_clock_mhz", "power_w")
                      if any(r[key] is not None for r in rounds)}
    rec["summary"]["qps"] = B / (rec["summary"]["ms_step"]["median"] / 1000.0)
    rec["rounds"] = rounds
    for _ in range(args.warmup):
        step()
    rec["kernels"] = kernel_breakdown(torch, step, args.profile_steps)
    ix.close()
    with open(os.path.join(args.out, "rerank_overlap.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps({key: v for key, v in rec.items() if key != "rounds"}), flush=True)


if __name__ == "__main__":
    main()
