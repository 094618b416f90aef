"""Per-phase cycle breakdown of the prefilter scan kernel (DESIGN.md sections 5, 5b, 5c): where a corpus tile's clocks go,
and so whether a change to the operand feed (e.g. a query tile kept resident in shared memory) can pay off.

    python tools/bench_prefilter_resident.py --out DIR [--rows 10000000] [--steps 10] [--c4-rows 5000000]

1. Builds the C2 index (brute-force cosine top-10, 10M x 768 f32, B = 1024) with bench.py's seeds.  For the s8 and the f16
   form of the prefilter: the scan kernel's ms (cdb_index_scan_ms_history, uninstrumented steps), candidates per query,
   the SM clock, and then the clock64 sums of the instrumented kernel (cdb_debug_scan_profile) as clocks per corpus tile
   and warpgroup.
2. The same for the u8 wgmma form (KIND 1) on bench.py's C4 secondary: quaternary dot product 5M x 1024, B 4096.
Records the card, its power limit and its SM clock in the same run.  Writes DIR/prefilter_resident.json and prints it.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED_CORPUS = 0xC05DA7A + 2     # bench.py
SEED_QUERY = 0xC05DA7A + 102
SEED_C4, SEED_C4_QUERY = 0xC05DA7A + 4, 0xC05DA7A + 104

# the TS_PROF_* slots of cdb_debug_scan_profile (csrc/tensor_scan.cu)
SLOTS = ["full_wait", "mma", "epilogue", "refresh", "empty_wait", "drift", "tiles", "consumer", "producer", "ctas", "math_wait",
         "epi_thr", "epi_fold", "epi_emit", "bound_rounds", "epi_cmax"]


def gpu_query(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    return [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else None


def scan_profile(enable):
    """switches the instrumented scan kernel on or off, returns the sums accumulated since the previous call"""
    from cosdata_b200 import _lib
    lib = _lib.load()
    fn = lib.cdb_debug_scan_profile
    fn.argtypes, fn.restype = [C.c_int32, C.POINTER(C.c_uint64)], C.c_int32
    out = (C.c_uint64 * len(SLOTS))()
    assert fn(1 if enable else 0, out) == 0
    return dict(zip(SLOTS, [int(v) for v in out]))


def per_tile(p):
    """consumer phases per tile and warpgroup, producer phases per tile (the producer issues every tile once per CTA).
    math_wait: the s8 kernel's warpgroups waiting for their turn at the tensor pipe (0 for the other forms).
    s8 kernel: epi_thr / epi_cmax / epi_fold / epi_emit split the epilogue (threshold, class maxima and hit test, per-class
    fold, emission), refresh is the bound warp's clocks in its rounds, bound_rounds its rounds per corpus tile of a CTA"""
    t = max(p["tiles"], 1)
    r = {k: p[k] / t for k in ("full_wait", "mma", "epilogue", "refresh", "consumer", "math_wait", "epi_thr", "epi_cmax", "epi_fold",
                                "epi_emit")}
    r.update({k: 2 * p[k] / t for k in ("empty_wait", "drift", "producer", "bound_rounds")})
    return r


def profile(ix, step, steps, scans_per_step):
    """scan kernel ms per step (uninstrumented kernel), then the instrumented kernel's clocks over two more steps"""
    import torch
    scan_profile(False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    for _ in range(steps):
        step()
    clk = gpu_query("clocks.sm")
    torch.cuda.synchronize()
    kern = ix.scan_ms_history(steps * scans_per_step)
    rec = {"kernel_ms": float(np.sum(kern)) / steps, "sm_clock_mhz": float(clk[0]) if clk else None}
    scan_profile(True)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    prof = scan_profile(False)
    rec["profile_sums"] = prof
    rec["clocks_per_tile"] = per_tile(prof)
    return rec


def c2(args):
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

    res, outs = {}, {}
    for name, form in (("s8", "1"), ("f16", "0")):
        os.environ["CDB_TS_S8"] = form
        r = profile(ix, step, args.steps, 1)
        cand = ix.last_candidate_counts(B)
        r["cand_mean"] = float(cand.mean())
        r["tops"] = 2.0 * n * dim * B / (r["kernel_ms"] * 1e-3) / 1e12
        res[name] = r
        outs[name] = (d_ids.cpu().numpy().copy(), d_scores.cpu().numpy().view(np.uint32).copy(), d_counts.cpu().numpy().copy())
        print(json.dumps({name: r}), flush=True)
    os.environ.pop("CDB_TS_S8", None)
    res["outputs_bit_identical"] = all(np.array_equal(a, b) for a, b in zip(outs["s8"], outs["f16"]))
    ix.close()
    return res


def c4(args):
    import torch
    import cosdata_b200 as cdb
    n, dim, B, k = args.c4_rows, 1024, 4096, 10
    ix = cdb.DenseIndex(dim=dim, storage_type=cdb.StorageType.SubByte2, metric=cdb.DistanceMetricKind.DotProduct, capacity=n)
    ix.append_synthetic(SEED_C4, n)
    dev = torch.device("cuda", 0)
    d_q = torch.from_numpy(cdb.synth_matrix(SEED_C4_QUERY, B, dim)).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream, mode=cdb.SearchMode.BRUTE_CODES)

    r = profile(ix, step, args.steps, (B + 2047) // 2048)   # one scan per chunk of <= 2048 queries
    r["tops"] = 2.0 * n * dim * B / (r["kernel_ms"] * 1e-3) / 1e12
    res = {"u8": r}
    print(json.dumps(res), flush=True)
    ix.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--c4-rows", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = gpu_query("name,power.limit,clocks.max.sm")
    rec = {"gpu": info[0] if info else None, "power_limit_w": info[1] if info else None,
           "max_sm_clock_mhz": info[2] if info else None}
    rec["c2"] = c2(args)
    rec["c4"] = c4(args)
    with open(os.path.join(args.out, "prefilter_resident.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
