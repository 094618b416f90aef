"""A/B of the prefilter's two forms (fp16 and s8, DESIGN.md section 5c) on the headline workload, and optionally of
bench.py between two builds.

    python tools/bench_prefilter_s8.py --out DIR [--rounds 5] [--steps 20] [--warmup 5] [--base-tree PATH] [--bench-runs 2]

1. Builds the C2 index (brute-force cosine top-10, 10M x 768 f32, B = 1024) with bench.py's seeds and alternates
   CDB_TS_S8=0 / 1 on it for --rounds rounds each: ms per step (CUDA events around --steps device searches), the prefilter
   kernel's ms (cdb_index_scan_ms_history), candidates per query, the SM clock during the round, and a bit-for-bit
   comparison of the two forms' outputs.  The achieved rate 2*N*D*B / kernel time is set against the measured integer and
   f16 tensor peaks (cdb.tensor_peak; s8 and u8 MMAs issue at the same rate).
2. With --base-tree (a built checkout of another commit): runs `bench.py --gpus 1` there and here, alternating, each with
   --dump-outputs, and compares the headline values and the dumped outputs.
Writes DIR/prefilter_s8.json and prints it.
"""
import argparse
import json
import os
import re
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


def ab_forms(args):
    import torch
    import cosdata_b200 as cdb
    n, dim, B, k = args.rows, 768, 1024, 10
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append_synthetic(SEED_CORPUS, n)
    dev = torch.device("cuda", 0)
    d_q = torch.from_numpy(cdb.synth_matrix(SEED_QUERY, B, dim)).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream)

    res = {"0": [], "1": []}
    outs = {}
    for rnd in range(args.rounds):
        for form in ("0", "1"):
            os.environ["CDB_TS_S8"] = form
            s8_before = ix.stats()["s8_searches"]
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                step()
            e1.record(stream)
            clk = gpu_query("clocks.sm")
            torch.cuda.synchronize()
            st = ix.stats()
            assert (st["s8_searches"] - s8_before > 0) == (form == "1"), ("the forced form did not run", form, st)
            assert st["fallback_queries"] == 0
            cand = ix.last_candidate_counts(B)
            kern = ix.scan_ms_history(args.steps)
            res[form].append({"ms_step": e0.elapsed_time(e1) / args.steps, "kernel_ms": float(np.median(kern)),
                              "cand_mean": float(cand.mean()), "cand_max": int(cand.max()),
                              "sm_clock_mhz": float(clk[0]) if clk else None})
            o = (d_ids.cpu().numpy().copy(), d_scores.cpu().numpy().view(np.uint32).copy(), d_counts.cpu().numpy().copy())
            if form in outs:
                assert all(np.array_equal(a, b) for a, b in zip(outs[form], o)), "a form's output changed between rounds"
            outs[form] = o
    os.environ.pop("CDB_TS_S8", None)
    identical = all(np.array_equal(a, b) for a, b in zip(outs["0"], outs["1"]))
    flop = 2.0 * n * dim * B
    peak_i8, _ = cdb.tensor_peak(True)
    peak_f16, _ = cdb.tensor_peak(False)
    summary = {}
    for form, name, peak in (("0", "f16", peak_f16), ("1", "s8", peak_i8)):
        km = stats([r["kernel_ms"] for r in res[form]])
        summary[name] = {"ms_step": stats([r["ms_step"] for r in res[form]]), "kernel_ms": km,
                         "cand_mean": stats([r["cand_mean"] for r in res[form]]),
                         "cand_max": max(r["cand_max"] for r in res[form]),
                         "sm_clock_mhz": stats([r["sm_clock_mhz"] for r in res[form] if r["sm_clock_mhz"] is not None] or [0]),
                         "achieved_tops": flop / (km["median"] * 1e-3) / 1e12,
                         "probe_peak_tops": peak, "share_of_probe_peak": flop / (km["median"] * 1e-3) / 1e12 / peak}
    summary["speedup_ms_step"] = summary["f16"]["ms_step"]["median"] / summary["s8"]["ms_step"]["median"]
    summary["outputs_bit_identical"] = bool(identical)
    ix.close()
    return {"rounds": res, "summary": summary}


def run_bench(tree, out_dir, args):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.bench_steps), "--warmup", str(args.bench_warmup),
           "--dump-outputs", out_dir]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, timeout=3000)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not line:
        return {"rc": r.returncode, "tail": (r.stdout + r.stderr)[-2000:]}
    j = json.loads(line[-1])
    return {"rc": 0, "value": j.get("value"), "unit": j.get("unit"), "secondary_errors": re.findall(r'"error": "[^"]*"', line[-1])}


def same_dumps(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    return fa == fb and all(np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f))) for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--base-tree", default=None)
    ap.add_argument("--bench-runs", type=int, default=2)
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--bench-warmup", type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = gpu_query("name,power.limit,clocks.max.sm")
    rec = {"gpu": info[0] if info else None, "power_limit_w": info[1] if info else None,
           "max_sm_clock_mhz": info[2] if info else None}
    rec["forms"] = ab_forms(args)
    print(json.dumps(rec["forms"]["summary"]), flush=True)
    if args.base_tree:
        runs = []
        for i in range(args.bench_runs):
            for name, tree in (("base", args.base_tree), ("branch", ROOT)):
                d = os.path.join(os.path.abspath(args.out), f"dump_{name}_{i}")
                r = run_bench(tree, d, args)
                r.update(tree=name, dump=d)
                runs.append(r)
                print(json.dumps(r), flush=True)
        vals = {n: [r["value"] for r in runs if r["tree"] == n and r.get("value")] for n in ("base", "branch")}
        rec["bench"] = {"runs": runs, "base": stats(vals["base"]) if vals["base"] else None,
                        "branch": stats(vals["branch"]) if vals["branch"] else None,
                        "dumps_identical": all(same_dumps(runs[0]["dump"], r["dump"]) for r in runs[1:])}
        if vals["base"] and vals["branch"]:
            rec["bench"]["speedup"] = float(np.median(vals["branch"]) / np.median(vals["base"]))
    with open(os.path.join(args.out, "prefilter_s8.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps({k: v for k, v in rec.items() if k != "forms"} | {"summary": rec["forms"]["summary"]}), flush=True)


if __name__ == "__main__":
    main()
