#!/usr/bin/env python
"""bench.py -- queries/s of the brute-force cosine hot path on H100 (BASELINE.json configs[1]).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA path
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port)
    python bench.py --steps K --dump-outputs DIR             # + the last timed step's results as DIR/<name>.npy

A "step" is one batch search of B=1024 queries over the whole resident corpus
(10M x 768 fp32 at N=1).  `value` is measured with every input already in HBM
(cdb_search_batch_device); `e2e` is the same step through cdb_search_batch with
HOST query/result buffers, copies inside the timed region.  For N>1 the corpus is
row-sharded over the ranks (strong scaling: the same 10M rows and the same queries),
each rank searches its shard, the per-shard top-k are all-gathered (NCCL) and merged
on every rank by cdb_merge_topk_device.

The reference arm times the CPU oracle (bit-faithful C/AVX2 port of the Rust path;
the Rust crate cannot be built in this image) on all host cores over a bounded
sample (a 1/8-size corpus shard, few queries) and scales linearly in rows.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SEED_CORPUS = 0xC05DA7A + 2
SEED_QUERY = 0xC05DA7A + 102
# NVIDIA H100 SXM data sheet (700 W): HBM3 bandwidth and dense f16/bf16 tensor rate -- roofline denominators when no
# measured peak is at hand; never reported as reached
H100_HBM_GBS = 3350.0
H100_F16_TFLOPS = 989.0


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir, **arrays):
    """arrays -> out_dir/<name>.npy, float32 / float64 only, at most DUMP_LIMIT_BYTES in all (checked before anything is
    written).  The callers pass what the timed path returned in its last step: ids and counts as float64 (exact for u32),
    scores as float32."""
    for name, a in arrays.items():
        if a.dtype not in (np.float32, np.float64):
            raise ValueError(f"dump_outputs: {name} is {a.dtype}, not float32 / float64")
    total = sum(a.nbytes for a in arrays.values())
    if total > DUMP_LIMIT_BYTES:
        raise ValueError(f"dump_outputs: {total} bytes exceed the {DUMP_LIMIT_BYTES}-byte limit")
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), a)


def dump_device_results(args, d_ids, d_scores, d_counts):
    """--dump-outputs: the device result buffers of the last timed step (ids [B][k] u32 as float64, scores f32, counts)"""
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, ids=d_ids.cpu().numpy().view(np.uint32).astype(np.float64),
                     scores=d_scores.cpu().numpy().astype(np.float32), counts=d_counts.cpu().numpy().astype(np.float64))


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--exact-only", action="store_true", help="pure FFMA scan (no tensor-core prefilter)")
    ap.add_argument("--cpu-sample-rows", type=int, default=1_250_000)
    ap.add_argument("--cpu-sample-queries", type=int, default=0, help="0 = max(16, host cores): one query per host thread like rayon")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the secondary records (other BASELINE.json shapes) of the N=1 line")
    ap.add_argument("--workload", default="c2", choices=["c2", "c3", "c4", "c5", "hnsw"],
                    help="c2 (default, the headline): brute cosine 10Mx768 f32; c4: quaternary inner product 50Mx1024, batch 4096; "
                         "hnsw: HNSW f16 search on a prebuilt graph (bench_data/, tools/build_hnsw_graph.py)")
    ap.add_argument("--ef", type=int, default=128)
    ap.add_argument("--hnsw-prof", action="store_true", help="c3: add the per-phase clock64 breakdown of one search (instrumented kernel variant)")
    ap.add_argument("--storage", default="f16", choices=["f16", "bf16"],
                    help="c3: f16 = the reference's HalfPrecisionFP (parity arm); bf16 = the labelled extension CDB_ST_BF16 (BASELINE.json's wording)")
    ap.add_argument("--hnsw-flags", type=int, default=None, help="c3: kernel variant flags (cdb_debug_set_hnsw_flags) for the timed steps")
    ap.add_argument("--hnsw-variants", action="store_true", help="c3: time every kernel variant (cdb_debug_set_hnsw_flags) on the same graph")
    ap.add_argument("--dump-ids", default=None, help="c3: write the result ids/scores of the batch to this .npz (A/B runs)")
    ap.add_argument("--graph", default=os.path.join(ROOT, "bench_data", "hnsw_100k_128_f16.npz"))
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write what the last timed step returned (ids, scores and, on the GPU paths, counts of the whole batch) as "
                         "DIR/<name>.npy (float64 / float32, <= 64 MB); every workload and --impl reference honour it; the inputs "
                         "are seeded, so two builds can be compared output for output")
    return ap.parse_args()


# ----------------------------------------------------------------------------- clocks
class ClockSampler:
    """samples nvidia-smi (read-only queries) during the timed region"""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index, period_ms=50):
        self.gpu = gpu_index
        self.period_ms = period_ms
        self.proc = None
        self.lines = []
        self.stamps = []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.gpu), "-lms", str(self.period_ms)], stdout=subprocess.PIPE, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())
            self.stamps.append(time.perf_counter())

    def stop(self, t_from=None, t_to=None):
        """median SM clock and throttle reasons of the samples that arrived in [t_from, t_to + one period] (host clock;
        a sample is printed at most one period after it was taken); without a window: every sample"""
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln, ts in zip(list(self.lines), list(self.stamps)):
            if t_from is not None and not (t_from <= ts <= t_to + self.period_ms / 1000.0):
                continue
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
            except ValueError:
                continue
            for nm, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def clock_sampling_repeats(total_ms, steps, warmup, min_load_ms=250.0, cap=2000):
    """untimed repeats of the step after the timed region so that warm-up + timed steps + repeats last ~min_load_ms
    (nvidia-smi delivers a sample every 20 ms).  A pure function of the MAX-REDUCED time of the timed region, i.e. the same
    integer on every rank: the repeats contain collectives, so a time-based loop per rank would deadlock."""
    per_step = max(float(total_ms) / max(int(steps), 1), 1e-3)
    missing = max(0.0, float(min_load_ms) - (int(steps) + int(warmup)) * per_step)
    return int(min(cap, missing / per_step + 0.999))


# ----------------------------------------------------------------------------- CPU baseline (oracle)
def cpu_queries(args):
    """the reference runs one query per rayon worker (indexes/mod.rs:268): give every host core a query"""
    cores = os.cpu_count() or 1
    return max(16, cores) if args.cpu_sample_queries <= 0 else args.cpu_sample_queries


def cpu_baseline(rows_full, dim, k, sample_rows, sample_queries, threads):
    """-> (qps scaled to the full corpus, seconds, description, (ids, scores) of the sample search for the parity gate)"""
    import oracle as orc
    sample_rows = min(sample_rows, rows_full)
    corpus = orc.synth_matrix(SEED_CORPUS, sample_rows, dim)
    queries = orc.synth_matrix(SEED_QUERY, sample_queries, dim)
    orc.brute_topk_f32(corpus[: min(sample_rows, 20000)], queries[:1], k, threads=threads)  # warm
    t0 = time.perf_counter()
    ids, scores = orc.brute_topk_f32(corpus, queries, k, threads=threads)
    dt = time.perf_counter() - t0
    qps_sample = sample_queries / dt
    qps_full = qps_sample * (sample_rows / rows_full)
    busy = min(threads, sample_queries)
    desc = (f"oracle port (C/AVX2+FMA), one query per thread like rayon: {sample_queries} queries on {busy} of {threads} host threads, "
            f"{sample_rows}x{dim} rows (1/{max(1, rows_full // sample_rows)} of the corpus) in {dt:.2f}s, scaled linearly in rows")
    # the 1-thread figure SURVEY 8d asks for: one query, one thread, a quarter of the sample rows (scaled like the rest)
    one = None
    try:
        r1 = max(1, sample_rows // 4)
        t1 = time.perf_counter()
        orc.brute_topk_f32(corpus[:r1], queries[:1], k, threads=1)
        d1 = time.perf_counter() - t1
        one = {"value": (1.0 / d1) * (r1 / rows_full), "unit": "queries/s", "sample": f"1 query on 1 thread, {r1}x{dim} rows in {d1:.2f}s"}
    except Exception:
        pass
    return qps_full, dt, desc, (ids, scores), busy, one


def run_reference(args, rank, world):
    if rank != 0:
        return
    threads = os.cpu_count() or 1
    import oracle as orc
    nqs = cpu_queries(args)
    sample_rows = min(args.cpu_sample_rows, args.rows)
    corpus = orc.synth_matrix(SEED_CORPUS, sample_rows, args.dim)
    queries = orc.synth_matrix(SEED_QUERY, nqs, args.dim)
    for _ in range(max(0, min(args.warmup, 1))):
        orc.brute_topk_f32(corpus[: min(sample_rows, 50000)], queries, args.k, threads=threads)
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        r_ids, r_scores = orc.brute_topk_f32(corpus, queries, args.k, threads=threads)
        times.append(time.perf_counter() - t0)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, ids=np.asarray(r_ids).view(np.uint32).astype(np.float64),
                     scores=np.asarray(r_scores).astype(np.float32))
    dt = float(np.sum(times))
    qps = args.steps * nqs / dt * (sample_rows / args.rows)
    busy = min(threads, nqs)
    sample = (f"each step = {nqs} queries (one per thread, {busy} of {threads} host threads busy) x {sample_rows}x{args.dim} rows "
              f"(1/{max(1, args.rows // sample_rows)} of the corpus), scaled linearly in rows")
    line = {
        "impl": "reference", "metric": "queries/sec, brute-force cosine top-10", "value": qps, "unit": "queries/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000.0 * dt / args.steps,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args, args.gpus),
        "cpu_baseline": {"value": qps, "unit": "queries/s", "cores": busy, "host_threads": threads, "kind": "port", "sample": sample},
        "e2e": {"value": qps, "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def workload_config(args, world):
    return {"workload": f"brute-force cosine top-{args.k}, {args.rows}x{args.dim} fp32 corpus, batch={args.batch} queries "
                        f"(BASELINE.json configs[1])",
            "rows": args.rows, "dim": args.dim, "batch": args.batch, "k": args.k,
            "sharding": f"rows/{world}" if world > 1 else "none", "l2": "inputs_exceed_l2 (corpus >> 50 MB)",
            "synthetic": "uniform[-1,1) counter RNG, include/cosdata_b200.h"}


# ----------------------------------------------------------------------------- our arm
def parity_abort(what):
    sys.stderr.write(f"bench.py: PARITY GATE FAILED: {what}\n")
    sys.stdout.flush()
    os._exit(3)


def run_ours(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    import cosdata_b200 as cdb
    from cosdata_b200.sharding import ShardGroup, shard_range

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the product path has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    row0, rows_local = shard_range(args.rows, world, rank)
    B, D, k = args.batch, args.dim, args.k

    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.FullPrecisionFP, metric=cdb.DistanceMetricKind.Cosine,
                        capacity=rows_local, device=local_rank, id_base=row0)
    # same global synthetic corpus for every world size: shard r holds rows [row0, row0+rows_local)
    ix.append_synthetic(SEED_CORPUS, rows_local, first_row=row0)

    # multi-GPU: the shard group behind the C ABI owns the NCCL communicator, the gather buffers and the merge
    # (csrc/shard_group.cu); torch.distributed only carries the 128-byte NCCL id to the other ranks and the barriers
    group = None
    if world > 1:
        box = [ShardGroup.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        group = ShardGroup.rank(box[0], world, rank, local_rank)
        group.attach(0, ix)

    q_host = cdb.synth_matrix(SEED_QUERY, B, D)
    d_q = torch.from_numpy(q_host).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)

    stream = torch.cuda.Stream(dev)   # a real (non-default) stream: the ABI treats NULL as "use the handle's own stream"
    torch.cuda.set_stream(stream)

    def step_device():
        if group is None:
            ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                                   stream.cuda_stream, exact_only=args.exact_only)
        else:   # local search -> ONE ncclAllGather of packed keys -> merge, all enqueued by one C call
            group.search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                                stream.cuda_stream, exact_only=args.exact_only)

    def step_e2e():
        # host queries in, host results out, through the public C-ABI call with HOST buffers (copies inside the call)
        if group is None:
            return ix.batch_search(q_host, k, exact_only=args.exact_only)[:2]
        return group.search(q_host, k, exact_only=args.exact_only)[:2]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    sampler = ClockSampler(local_rank, period_ms=20)   # started early: nvidia-smi needs ~0.1 s before its first sample
    sampler.start()
    # ---- parity gate BEFORE any timing (SURVEY 8d): the path that will be timed must return exactly what the exact scan
    # returns on the resident rows.  (At N = 1 the CPU oracle leg below adds an independent check.)
    gate_q = min(64, B)
    got_ids, got_scores, _, _ = ix.batch_search(q_host[:gate_q], k, exact_only=args.exact_only)
    ex_ids, ex_scores, _, _ = ix.batch_search(q_host[:gate_q], k, exact_only=True)
    if not (np.array_equal(got_ids, ex_ids) and np.array_equal(got_scores.view(np.uint32), ex_scores.view(np.uint32))):
        parity_abort("prefilter path differs from the exact scan on the resident shard")
    parity = {"prefilter_vs_exact_scan": {"queries": gate_q, "rows": rows_local, "bit_identical": True}}
    if group is not None:   # sharded merge against the same queries: every rank holds the merged result
        m_ids, m_scores = group.search(q_host[:gate_q], k, exact_only=args.exact_only)[:2]
        l_keys = None
        from cosdata_b200.sharding import pack_keys, merge_packed
        mine = torch.from_numpy(pack_keys(ex_ids, ex_scores).view(np.int64)).to(dev)
        allk = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allk, mine)
        w_ids, w_scores, _ = merge_packed(np.stack([t.cpu().numpy().view(np.uint64) for t in allk]), k)
        if not (np.array_equal(m_ids, w_ids) and np.array_equal(m_scores.view(np.uint32), w_scores.view(np.uint32))):
            parity_abort("sharded search differs from the merge of the per-shard exact scans")
        parity["sharded_vs_merged_exact_scans"] = {"queries": gate_q, "shards": world, "bit_identical": True}

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        barrier()
        l0 = cdb.kernel_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        barrier()
        launches = cdb.kernel_launch_count() - l0
        ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), launches

    def timed_host(fn, steps, warmup):
        """host-blocking calls: wall clock between barriers (the call returns when the results are in host memory)"""
        for _ in range(warmup):
            fn()
        barrier()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize(dev)
        ms = torch.tensor([(time.perf_counter() - t0) * 1000.0], dtype=torch.float64, device=dev)
        barrier()
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    t_from = time.perf_counter()
    total_ms, launches_timed = timed(step_device, args.steps, max(args.warmup, 3))
    if rank == 0:    # the results of the last timed step, before anything else touches the buffers
        dump_device_results(args, d_ids, d_scores, d_counts)
    # nvidia-smi delivers a sample every 20 ms: a timed region shorter than ~0.2 s is followed by UNTIMED repeats of the
    # same step so that the clock record still comes from this load (the timing above is not affected)
    # (the number of repeats is derived from the max-reduced step time, so every rank issues the same number of collectives)
    scan_ms = ix.scan_ms_history(args.steps)      # the dominant kernel's launches of the TIMED steps
    extra = clock_sampling_repeats(total_ms, args.steps, max(args.warmup, 3))
    for _ in range(extra):
        step_device()
    barrier()
    t_to = time.perf_counter()
    clocks = sampler.stop(t_from, t_to)
    clocks["window"] = "warm-up + timed steps" + (f" + {extra} untimed repeats (~0.25 s of load)" if extra else "")
    e2e_ms = timed_host(step_e2e, args.steps, 2)

    value = args.steps * B / (total_ms / 1000.0)
    e2e_value = args.steps * B / (e2e_ms / 1000.0)

    # roofline of the dominant kernel (DESIGN.md section 6).  Algorithmic work per launch:
    #   flops = 2*rows*D*B ; bytes = rows*(D*4+4) + B*D*4 (fp32 corpus) -- the wgmma prefilter reads the
    #   fp16 shadow instead (rows*D*2 bytes), reported as shadow_bytes.
    stats = ix.stats()
    tensor_path = stats["tensor_searches"] > 0 and stats["fallback_queries"] == 0
    alg_bytes = rows_local * (D * 4 + 4) + B * D * 4
    alg_flops = 2.0 * rows_local * D * B
    peaks = _peaks()
    peak_src = "measured (MEASURED_PEAKS.json)" if "hbm_gbs" in peaks else f"H100 SXM data sheet ({H100_HBM_GBS:.0f} GB/s, {H100_F16_TFLOPS:.0f} TFLOP/s dense f16)"
    hbm_peak = float(peaks.get("hbm_gbs", H100_HBM_GBS))
    tc_peak = float(peaks.get("bf16_tflops", H100_F16_TFLOPS))
    scan_avg_ms = float(np.mean(scan_ms)) if len(scan_ms) else float("nan")
    traffic, traffic_src = None, None
    if tensor_path:
        achieved = alg_flops / (scan_avg_ms / 1000.0) / 1e12
        cand = ix.last_candidate_counts(B)
        roofline = {"bound": "tensor", "achieved": achieved, "peak": tc_peak, "unit": "TFLOP/s", "frac": achieved / tc_peak,
                    "traffic": traffic, "traffic_source": traffic_src, "peak_source": peak_src + ", dense bf16/fp16 burst",
                    "kernel": "tensor_scan_kernel (wgmma fp16 prefilter, threshold epilogue)", "kernel_ms": scan_avg_ms,
                    "alg_flops_per_launch": alg_flops, "shadow_bytes_per_launch": rows_local * D * 2,
                    "hbm_gbs_on_shadow": rows_local * D * 2 / (scan_avg_ms / 1000.0) / 1e9,
                    "candidates_per_query": {"mean": float(cand.mean()), "max": int(cand.max())},
                    "note": "candidates are re-scored exactly (rerank_f32_kernel); final ids/scores are bit-identical to the exact scan"}
    else:
        achieved = alg_bytes / (scan_avg_ms / 1000.0) / 1e9
        roofline = {"bound": "hbm", "achieved": achieved, "peak": hbm_peak, "unit": "GB/s", "frac": achieved / hbm_peak,
                    "traffic": traffic, "traffic_source": traffic_src, "peak_source": peak_src,
                    "kernel": "scan_f32_kernel (exact FFMA scan, fused top-k)", "kernel_ms": scan_avg_ms,
                    "alg_bytes_per_launch": alg_bytes, "fp32_tflops": alg_flops / (scan_avg_ms / 1000.0) / 1e12,
                    "note": "HBM-bound only for small per-pass batches; at large B the exact FP32 scan is FFMA/L2-bound"}

    line = {
        "metric": "queries/sec, brute-force cosine top-10", "value": value, "unit": "queries/s", "n_gpus": world,
        "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": total_ms / args.steps,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args, world), "clocks": clocks,
        "e2e": {"value": e2e_value, "unit": "queries/s", "h2d_bytes_per_step": B * D * 4, "d2h_bytes_per_step": B * k * 8 + B * 5,
                "ms_per_step": e2e_ms / args.steps, "timing": "host wall clock around the blocking C-ABI call, max over ranks"},
        "gpu_launches": int(launches_timed), "roofline": roofline, "parity_checked": parity,
    }
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        threads = os.cpu_count() or 1
        nqs = cpu_queries(args)
        v, dt, sample, (o_ids, o_scores), busy, one = cpu_baseline(args.rows, D, k, args.cpu_sample_rows, nqs, threads)
        line["cpu_baseline"] = {"value": v, "unit": "queries/s", "cores": busy, "host_threads": threads, "kind": "port", "sample": sample,
                                "one_thread": one}
        # oracle leg of the parity gate: the same sample (rows [0, sample_rows) x nqs queries) through the CUDA path
        srows = min(args.cpu_sample_rows, args.rows)
        sm = cdb.DenseIndex(dim=D, capacity=srows, device=local_rank)
        sm.append_synthetic(SEED_CORPUS, srows)
        g_ids, g_scores, _, _ = sm.batch_search(cdb.synth_matrix(SEED_QUERY, nqs, D), k, exact_only=args.exact_only)
        took_tensor = sm.stats()["tensor_searches"] > 0
        sm.close()
        if not (np.array_equal(g_ids, o_ids) and np.array_equal(g_scores.view(np.uint32), o_scores.view(np.uint32))):
            parity_abort("CUDA path differs from the CPU oracle on the sample shard")
        line["parity_checked"]["cuda_vs_cpu_oracle"] = {"queries": nqs, "rows": srows, "bit_identical": True, "tensor_path": took_tensor}
        line["recall_at_10"] = float(np.mean([len(set(g_ids[i]) & set(o_ids[i])) / k for i in range(nqs)]))
        line["recall_note"] = "computed in this run: CUDA top-10 vs the CPU oracle's exact top-10 on the sample shard"
    if rank == 0 and world == 1 and not args.no_secondary:
        try:
            line["secondary"] = secondary_records(args, ix, cdb, torch, stream, dev, q_host)
        except Exception as e:            # a secondary record must never take the headline down
            line["secondary"] = [{"error": repr(e)}]
    if rank == 0:
        print(json.dumps(line), flush=True)
    if group is not None:
        group.close()
    ix.close()
    if world > 1:
        dist.destroy_process_group()


def secondary_records(args, ix, cdb, torch, stream, dev, q_host):
    """small, fast extra measurements on the same box (each < ~2 s): the other BASELINE.json shapes the driver cannot run
    separately, with their own rooflines and clock samples"""
    out = []
    pk = _peaks()
    hbm = float(pk.get("hbm_gbs", H100_HBM_GBS))
    B, D, k, rows = args.batch, args.dim, args.k, ix.size

    def run(fn, n, flush=None):
        torch.cuda.synchronize()
        sam = ClockSampler(dev.index, period_ms=20)
        sam.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if flush is None:
            e0.record(stream)
            for _ in range(n):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n
        else:                      # cold: L2 flushed before every launch, each launch timed on its own
            tot = 0.0
            for _ in range(n):
                flush()
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                tot += e0.elapsed_time(e1)
            ms = tot / n
        return ms, sam.stop()

    d_q = torch.from_numpy(q_host).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_sc = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_cn = torch.empty((B,), dtype=torch.int32, device=dev)
    # ---- the headline corpus at small batches: HBM-bound (north_star: ">= 70 % of the HBM roofline on batched cosine")
    for nb_, exact in ((1, True), (8, True), (8, False)):
        def fn():
            ix.batch_search_device(d_q.data_ptr(), nb_, k, d_ids.data_ptr(), d_sc.data_ptr(), d_cn.data_ptr(), None,
                                   stream.cuda_stream, exact_only=exact)
        for _ in range(3):
            fn()
        nl_ = 50 if exact else 150        # >= ~0.3 s of back-to-back launches so that nvidia-smi gets samples
        ms, clk = run(fn, nl_)
        kms = float(np.mean(ix.scan_ms_history(50)))
        f32_bytes = rows * (D * 4 + 4) + nb_ * D * 4
        sh_bytes = rows * D * 2 + nb_ * D * 2
        alg = f32_bytes if exact else sh_bytes
        out.append({"name": f"brute-force cosine {rows}x{D}, batch={nb_}, " + ("exact f32 scan" if exact else "fp16 prefilter + exact re-rank"),
                    "value": nb_ / (ms / 1000.0), "unit": "queries/s", "ms_per_step": ms, "launches_timed": nl_, "clocks": clk,
                    "roofline": {"bound": "hbm", "achieved": alg / (kms / 1000.0) / 1e9, "peak": hbm, "unit": "GB/s",
                                 "frac": alg / (kms / 1000.0) / 1e9 / hbm, "kernel_ms": kms, "alg_bytes_per_launch": alg,
                                 "peak_note": "peak = measured device copy (read + write); a read-only stream can exceed it slightly",
                                 "kernel": "scan_f32_kernel (f32 rows)" if exact else "tensor_scan_kernel (fp16 shadow rows)"}})
    # ---- BASELINE.json configs[0]: 100k x 128 fp32, batch = 1 (the reference's own CPU-runnable case), warm and cold L2
    c1 = cdb.DenseIndex(dim=128, capacity=100_000, device=dev.index)
    c1.append_synthetic(0xC05DA7A + 1, 100_000)
    q1 = torch.from_numpy(cdb.synth_matrix(0xC05DA7A + 101, 1, 128)).to(dev)

    def fn1():
        c1.batch_search_device(q1.data_ptr(), 1, k, d_ids.data_ptr(), d_sc.data_ptr(), d_cn.data_ptr(), None, stream.cuda_stream)
    for _ in range(5):
        fn1()
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    warm_ms, clk_w = run(fn1, 200)
    cold_ms, clk_c = run(fn1, 30, flush=lambda: scratch.zero_())
    c1.close()
    del scratch
    c1_bytes = 100_000 * (128 * 4 + 4) + 128 * 4
    out.append({"name": "brute-force cosine 100000x128 fp32, batch=1 (BASELINE.json configs[0])", "value": 1000.0 / warm_ms,
                "unit": "queries/s", "ms_per_step": warm_ms, "cold_l2_ms_per_step": cold_ms, "clocks": clk_w,
                "roofline": {"bound": "hbm", "achieved": c1_bytes / (cold_ms / 1000.0) / 1e9, "peak": hbm, "unit": "GB/s",
                             "frac": c1_bytes / (cold_ms / 1000.0) / 1e9 / hbm, "alg_bytes_per_launch": c1_bytes,
                             "note": "51 MB per query: warm = L2-resident + launch latency bound; cold = L2 flushed (256 MB write) before every launch, "
                                     "whole step timed (quantize + scan + merge launches), so the HBM fraction is a latency figure"}})
    # ---- BASELINE.json configs[3] on a 5M shard: quaternary inner product, batch 4096, exact integer scores on wgmma u8
    try:
        i8_tops, _ = cdb.tensor_peak(True, dev.index)
        f16_tops, _ = cdb.tensor_peak(False, dev.index)
        r4, D4, B4 = 5_000_000, 1024, 4096
        c4 = cdb.DenseIndex(dim=D4, storage_type=cdb.StorageType.SubByte2, metric=cdb.DistanceMetricKind.DotProduct, capacity=r4, device=dev.index)
        c4.append_synthetic(0xC05DA7A + 4, r4)
        q4 = torch.from_numpy(cdb.synth_matrix(0xC05DA7A + 104, B4, D4)).to(dev)
        i4 = torch.empty((B4, k), dtype=torch.int32, device=dev)
        s4 = torch.empty((B4, k), dtype=torch.float32, device=dev)
        n4 = torch.empty((B4,), dtype=torch.int32, device=dev)

        def fn4():
            c4.batch_search_device(q4.data_ptr(), B4, k, i4.data_ptr(), s4.data_ptr(), n4.data_ptr(), None, stream.cuda_stream,
                                   mode=cdb.SearchMode.BRUTE_CODES)
        for _ in range(2):
            fn4()
        ms4, clk4 = run(fn4, 5)
        kms4 = float(np.sum(c4.scan_ms_history(5 * ((B4 + 2047) // 2048)))) / 5
        ops4 = 2.0 * r4 * D4 * B4
        st4 = c4.stats()
        c4.close()
        out.append({"name": f"quaternary-quantized inner product {r4}x{D4}, batch={B4} (BASELINE.json configs[3] on a 1/10 shard)",
                    "value": B4 / (ms4 / 1000.0), "unit": "queries/s", "ms_per_step": ms4, "clocks": clk4,
                    "roofline": {"bound": "tensor", "achieved": ops4 / (kms4 / 1000.0) / 1e12, "peak": i8_tops, "unit": "TOP/s",
                                 "frac": ops4 / (kms4 / 1000.0) / 1e12 / i8_tops, "kernel_ms": kms4, "alg_ops_per_launch": ops4,
                                 "peak_source": "measured in this run: dense wgmma u8 issue-rate probe (csrc/tc_probe.cu); "
                                                f"the same probe with f16 gives {f16_tops:.0f} TFLOP/s next to the cuBLAS bf16 "
                                                f"{float(pk.get('bf16_tflops', 0)):.0f}",
                                 "kernel": "tensor_scan_kernel<KIND=1> (wgmma u8, exact)", "tensor_path": st4}})
    except Exception as e:
        out.append({"name": "quaternary-quantized inner product (configs[3] shard)", "error": repr(e)})
    # ---- BASELINE.json configs[2] at 1/10 size: HNSW f16, ef_search 128, batch 1024; graph built on the GPU (reference defaults)
    try:
        out.append(hnsw_record(cdb, torch, dev, stream, 1_000_000, 768, 1024, k, 128, hbm))
    except Exception as e:
        out.append({"name": "HNSW dense index (configs[2] at 1M rows)", "error": repr(e)})
    return out


def hnsw_record(cdb, torch, dev, stream, rows, D, B, k, ef, hbm):
    """clustered synthetic rows generated on device, graph built by cdb_index_build_graph (nbrs 32/64, ef_construction 128,
    9 layers), search timed over 10 batches, recall@k against the exact scan of the same rows"""
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    ncent = 4096
    centres = torch.randn((ncent, D), generator=g, device=dev)
    scale = 1.0 / (4.5 * 1.06)
    hx = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.HalfPrecisionFP, metric=cdb.DistanceMetricKind.Cosine,
                        capacity=rows + 1, device=dev.index, keep_raw_f32=True)
    for off in range(0, rows, 500_000):
        m = min(500_000, rows - off)
        idx = torch.randint(0, ncent, (m,), generator=g, device=dev)
        x = ((centres[idx] + 0.35 * torch.randn((m, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
        torch.cuda.synchronize()
        hx.append_device(x.data_ptr(), m)
        del x, idx
    idx = torch.randint(0, ncent, (B,), generator=g, device=dev)
    d_q = ((centres[idx] + 0.35 * torch.randn((B, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
    q_host = d_q.cpu().numpy()
    t0 = time.perf_counter()
    hx.build_graph(9, 32, 64, 128, 64, 4096, 7)
    torch.cuda.synchronize()
    t_build = time.perf_counter() - t0
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_sc = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_cn = torch.empty((B,), dtype=torch.int32, device=dev)

    def step():
        hx.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_sc.data_ptr(), d_cn.data_ptr(), None, stream.cuda_stream,
                               mode=cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64)
    ev0, pp0 = hx.hnsw_counters()
    step()
    torch.cuda.synchronize()
    ev1, pp1 = hx.hnsw_counters()
    sam = ClockSampler(dev.index, period_ms=20)
    sam.start()
    for _ in range(10):
        step()                              # nvidia-smi needs ~0.1 s before its first sample
    torch.cuda.synchronize()
    t_from = time.perf_counter()
    ms = _timed_single(step, 60, 3, stream) / 60
    clk = sam.stop(t_from, time.perf_counter())
    kms = float(np.mean(hx.scan_ms_history(60)))
    ids = d_ids.cpu().numpy().view(np.uint32)
    gt = hx.batch_search(q_host, k + 1, cdb.SearchMode.BRUTE_RAW)[0]
    gt = [[i for i in row if i != rows][:k] for row in gt]
    recall = float(np.mean([len(set(ids[i]) & set(gt[i])) / k for i in range(B)]))
    hx.close()
    evals, pops = ev1 - ev0, pp1 - pp0
    alg = evals * (D * 2 + 4) + pops * 64 * 4
    return {"name": f"HNSW dense index {rows}x{D} f16, ef_search={ef}, batch={B} (BASELINE.json configs[2] at 1/10 of the rows; "
                    "graph built on the GPU with the reference defaults)",
            "value": B / (ms / 1000.0), "unit": "queries/s", "ms_per_step": ms, "clocks": clk, "recall_at_10": recall,
            "build_seconds": t_build,
            "roofline": {"bound": "hbm", "achieved": alg / (kms / 1000.0) / 1e9, "peak": hbm, "unit": "GB/s",
                         "frac": alg / (kms / 1000.0) / 1e9 / hbm, "kernel_ms": kms, "alg_bytes_per_launch": alg,
                         "evals_per_query": evals / B, "pops_per_query": pops / B,
                         "kernel": "hnsw_search_warp_kernel (random row gathers; latency- not bandwidth-bound)"}}


# ----------------------------------------------------------------------------- secondary workloads (reporting modes)
def _timed_single(fn, steps, warmup, stream):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {}


def run_c4(args):
    """BASELINE.json configs[3]: quaternary-quantized inner product, 50M x 1024, batch 4096, 1 GPU"""
    import torch
    import cosdata_b200 as cdb
    rows = args.rows if args.rows != 10_000_000 else 50_000_000
    D = args.dim if args.dim != 768 else 1024
    B = args.batch if args.batch != 1024 else 4096
    k = args.k
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    seed_c, seed_q = 0xC05DA7A + 4, 0xC05DA7A + 104
    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.SubByte2, metric=cdb.DistanceMetricKind.DotProduct,
                        capacity=rows, device=0)
    ix.append_synthetic(seed_c, rows)
    q_host = cdb.synth_matrix(seed_q, B, D)
    d_q = torch.from_numpy(q_host).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream, mode=cdb.SearchMode.BRUTE_CODES, exact_only=args.exact_only)

    def step_e2e():
        ix.batch_search(q_host, k, cdb.SearchMode.BRUTE_CODES, exact_only=args.exact_only)

    sampler = ClockSampler(0)
    sampler.start()
    l0 = cdb.kernel_launch_count()
    ms = _timed_single(step, args.steps, max(args.warmup, 3), stream)
    dump_device_results(args, d_ids, d_scores, d_counts)
    clocks = sampler.stop()
    launches = (cdb.kernel_launch_count() - l0) * args.steps // (args.steps + max(args.warmup, 3))
    nchunks = (B + 2047) // 2048
    scan_ms = ix.scan_ms_history(args.steps * nchunks)
    e2e_ms = _timed_single(step_e2e, args.steps, 1, stream)
    st = ix.stats()
    kernel_ms = float(np.sum(scan_ms)) / args.steps
    ops = 2.0 * rows * D * B
    pk = _peaks()
    peak, _ = cdb.tensor_peak(True, 0)     # dense wgmma u8 issue-rate probe, measured in this run (csrc/tc_probe.cu)
    achieved = ops / (kernel_ms / 1000.0) / 1e12
    line = {
        "metric": "queries/sec, quaternary inner product top-10", "value": args.steps * B / (ms / 1000.0), "unit": "queries/s",
        "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "u8 digits -> s32 (exact)", "data": "synthetic",
        "config": {"workload": f"quaternary-quantized inner product, {rows}x{D}, batch={B} (BASELINE.json configs[3])",
                   "rows": rows, "dim": D, "batch": B, "k": k, "l2": "inputs_exceed_l2"},
        "clocks": clocks, "gpu_launches": int(launches),
        "e2e": {"value": args.steps * B / (e2e_ms / 1000.0), "unit": "queries/s", "h2d_bytes_per_step": B * D * 4,
                "d2h_bytes_per_step": B * k * 8 + B * 5, "ms_per_step": e2e_ms / args.steps},
        "roofline": {"bound": "tensor", "achieved": achieved, "peak": peak, "unit": "TOP/s", "frac": achieved / peak, "traffic": None,
                     "peak_source": "measured in this run: dense wgmma u8 issue-rate probe (cdb_debug_tensor_peak); cuBLAS bf16 in "
                                    f"MEASURED_PEAKS.json: {float(pk.get('bf16_tflops', 0)):.0f} TFLOP/s",
                     "kernel": "tensor_scan_kernel<KIND=1> (wgmma u8, exact)", "kernel_ms": kernel_ms,
                     "alg_ops_per_launch": ops, "digit_bytes": rows * D, "tensor_path": st},
        "recall_at_10": 1.0, "recall_note": "exact integer scores; ids identical to the CPU oracle (tests/test_gpu_tensor_u8.py)",
    }
    if not args.no_cpu_baseline:
        import oracle as orc
        threads = os.cpu_count() or 1
        srows = min(rows, 1_250_000)
        codes, mags = orc.quantize_batch(2, orc.synth_matrix(seed_c, 4096, D))   # warm the library
        t0 = time.perf_counter()
        corpus = orc.synth_matrix(seed_c, srows, D)
        cb = orc.code_bytes(2, D)
        codes = np.zeros((srows, cb), dtype=np.uint8)
        mags = np.zeros(srows, dtype=np.float32)
        from oracle.pyoracle import lib, _p
        L = lib()
        for i in range(srows):                       # quantize (not timed as search work)
            L.orc_quantize(2, -1.0, 1.0, corpus[i].ctypes.data, D, codes[i].ctypes.data, mags[i:i + 1].ctypes.data)
        qc, qm = orc.quantize_batch(2, q_host[:16])
        t1 = time.perf_counter()
        orc.brute_topk_codes(3, 2, D, codes, mags, qc, qm, k, threads=threads)
        dt = time.perf_counter() - t1
        v = 16 / dt * (srows / rows)
        line["cpu_baseline"] = {"value": v, "unit": "queries/s", "cores": threads, "kind": "port",
                                "sample": f"oracle dot_product_quaternary (AVX2) on {srows}x{D} codes x 16 queries in {dt:.2f}s, scaled linearly in rows"}
    print(json.dumps(line), flush=True)
    ix.close()


def run_hnsw(args):
    """HNSW f16 search (BASELINE.json configs[2] shape at the scale the CPU builder can produce): graph built by
    tools/build_hnsw_graph.py with the reference defaults, searched with ef_search = --ef"""
    import torch
    import cosdata_b200 as cdb
    import oracle as orc
    from oracle import pyhnsw
    z = np.load(args.graph)
    vecs, root = z["vecs"], z["root"]
    n, D = vecs.shape
    B, k = args.batch, args.k
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    node_row = [z[f"node_row{l}"] for l in range(10)]
    adj = [z[f"adj{l}"] for l in range(10)]
    child = [z[f"child{l}"] for l in range(10)]
    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.HalfPrecisionFP, metric=cdb.DistanceMetricKind.Cosine,
                        capacity=n + 1, device=0, keep_raw_f32=True)
    ix.append(np.concatenate([vecs, root[None]], axis=0))
    ix.set_graph(9, 32, 64, int(z["entry"]), n, node_row, adj, child)
    rng = np.random.default_rng(5)
    q_host = (vecs[rng.integers(0, n, B)] + 0.05 * rng.normal(size=(B, D))).astype(np.float32)
    d_q = torch.from_numpy(q_host).to(dev)
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream, mode=cdb.SearchMode.HNSW, ef_search=args.ef, shortlist_size=64)

    if args.hnsw_flags is not None:
        cdb.debug_set_hnsw_flags(args.hnsw_flags)
    sampler = ClockSampler(0, period_ms=20)
    sampler.start()
    ev0, pp0 = ix.hnsw_counters()
    step()
    torch.cuda.synchronize()
    ev1, pp1 = ix.hnsw_counters()
    evals, pops = ev1 - ev0, pp1 - pp0
    t_from = time.perf_counter()
    l0 = cdb.kernel_launch_count()
    ms = _timed_single(step, args.steps, max(args.warmup, 3), stream)
    dump_device_results(args, d_ids, d_scores, d_counts)
    launches = (cdb.kernel_launch_count() - l0) * args.steps // (args.steps + max(args.warmup, 3))
    scan_ms = ix.scan_ms_history(args.steps)
    while time.perf_counter() - t_from < 0.3:      # untimed repeats of the same step: the clock record needs ~0.2 s of this load
        step()
        torch.cuda.synchronize()
    clocks = sampler.stop(t_from, time.perf_counter())
    e2e_ms = _timed_single(lambda: ix.batch_search(q_host, k, cdb.SearchMode.HNSW, ef_search=args.ef, shortlist_size=64),
                           args.steps, 1, stream)
    ids = d_ids.cpu().numpy().view(np.uint32)
    # recall@10 against the exact top-10 (GPU exact scan over the same rows; rows 0..n-1, root excluded by id)
    ex = cdb.DenseIndex(dim=D, capacity=n, device=0)
    ex.append(vecs)
    gt, _, _, _ = ex.batch_search(q_host, k)
    ex.close()
    recall = float(np.mean([len(set(ids[i]) & set(gt[i])) / k for i in range(B)]))
    # parity + CPU baseline on a sample with the oracle (same graph)
    fg = pyhnsw.FlatGraph(orc.METRIC_COSINE, orc.ST_F16, D, *orc.quantize_batch(orc.ST_F16, np.concatenate([vecs, root[None]])),
                          n, 9, 32, 64, int(z["entry"]), node_row, adj, child)
    threads = os.cpu_count() or 1
    ns = min(B, 256)
    t0 = time.perf_counter()
    w = pyhnsw.search_batch(fg, vecs, q_host[:ns], k, ef_search=args.ef, threads=threads)
    dt = time.perf_counter() - t0
    parity = bool(np.array_equal(ids[:ns], w[0]) and np.array_equal(d_scores.cpu().numpy()[:ns].view(np.uint32), w[1].view(np.uint32)))
    orc_recall = float(np.mean([len(set(w[0][i]) & set(gt[i])) / k for i in range(ns)]))
    kernel_ms = float(np.mean(scan_ms))
    alg_bytes = evals * (D * 2 + 4) + pops * 64 * 4          # SURVEY 8d: evals*(D*s+4) + pops*(nbrs*4), counted on this graph
    pk = _peaks()
    hbm = float(pk.get("hbm_gbs", H100_HBM_GBS))
    ach = alg_bytes / (kernel_ms / 1000.0) / 1e9
    line = {
        "metric": "queries/sec + recall@10, HNSW f16", "value": args.steps * B / (ms / 1000.0), "unit": "queries/s", "n_gpus": 1,
        "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "f16 (f32 accumulate, reference order)", "data": "synthetic (clustered)",
        "config": {"workload": f"HNSW dense index, {n}x{D} f16, ef_search={args.ef}, batch={B} (BASELINE.json configs[2] shape; "
                               "graph built by the CPU oracle with the reference defaults)", "rows": n, "dim": D, "batch": B, "k": k},
        "clocks": clocks, "gpu_launches": int(launches),
        "e2e": {"value": args.steps * B / (e2e_ms / 1000.0), "unit": "queries/s", "h2d_bytes_per_step": B * D * 4,
                "d2h_bytes_per_step": B * k * 8 + B * 5, "ms_per_step": e2e_ms / args.steps},
        "roofline": {"bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm, "traffic": None,
                     "kernel": "hnsw_search_kernel (random row gathers)", "kernel_ms": kernel_ms, "alg_bytes_per_launch": alg_bytes,
                     "evals_per_query": evals / B, "pops_per_query": pops / B},
        "recall_at_10": recall, "oracle_recall_at_10": orc_recall, "parity_with_oracle_on_sample": parity,
        "cpu_baseline": {"value": ns / dt, "unit": "queries/s", "cores": threads, "kind": "port",
                         "sample": f"oracle ann_search + re-rank, {ns} queries, one query per thread, {dt:.2f}s"},
    }
    print(json.dumps(line), flush=True)
    ix.close()


def run_c3(args):
    """BASELINE.json configs[2]: HNSW dense index, 10M x 768 f16 ("bf16" in the JSON; the reference has IEEE f16 only),
    ef_search=128, batch=1024.  The graph is built ON THE GPU by cdb_index_build_graph with the reference defaults
    (nbrs 32/64, ef_construction 128, 9 layers); data = clustered synthetic rows generated on device with torch."""
    import torch
    import cosdata_b200 as cdb
    rows, D, B, k = args.rows, args.dim, args.batch, args.k
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    ncent = 4096
    centres = torch.randn((ncent, D), generator=g, device=dev)
    scale = 1.0 / (4.5 * 1.06)            # |x| < 1 with overwhelming probability; clamp below keeps the quantizer's domain
    st_ = cdb.StorageType.BFloat16 if args.storage == "bf16" else cdb.StorageType.HalfPrecisionFP
    ix = cdb.DenseIndex(dim=D, storage_type=st_, metric=cdb.DistanceMetricKind.Cosine,
                        capacity=rows + 1, device=0, keep_raw_f32=True)
    chunk = 500_000
    t0 = time.perf_counter()
    for off in range(0, rows, chunk):
        m = min(chunk, rows - off)
        idx = torch.randint(0, ncent, (m,), generator=g, device=dev)
        x = ((centres[idx] + 0.35 * torch.randn((m, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
        torch.cuda.synchronize()
        ix.append_device(x.data_ptr(), m)
        del x, idx
    t_load = time.perf_counter() - t0
    # queries: perturbed stored rows (generated the same way from a few row indices is not possible without keeping
    # the rows, so draw fresh points from the same mixture)
    idx = torch.randint(0, ncent, (B,), generator=g, device=dev)
    d_q = ((centres[idx] + 0.35 * torch.randn((B, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
    q_host = d_q.cpu().numpy()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ix.build_graph(9, 32, 64, 128, 64, 4096, 7)
    t_build = time.perf_counter() - t0
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)

    def step():
        ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                               stream.cuda_stream, mode=cdb.SearchMode.HNSW, ef_search=args.ef, shortlist_size=64)

    if args.hnsw_flags is not None:
        cdb.debug_set_hnsw_flags(args.hnsw_flags)
    sampler = ClockSampler(0, period_ms=20)
    sampler.start()
    ev0, pp0 = ix.hnsw_counters()
    step()
    torch.cuda.synchronize()
    ev1, pp1 = ix.hnsw_counters()
    evals, pops = ev1 - ev0, pp1 - pp0
    t_from = time.perf_counter()
    l0 = cdb.kernel_launch_count()
    ms = _timed_single(step, args.steps, max(args.warmup, 3), stream)
    dump_device_results(args, d_ids, d_scores, d_counts)
    launches = (cdb.kernel_launch_count() - l0) * args.steps // (args.steps + max(args.warmup, 3))
    scan_ms = ix.scan_ms_history(args.steps)
    while time.perf_counter() - t_from < 0.3:      # untimed repeats of the same step: the clock record needs ~0.2 s of this load
        step()
        torch.cuda.synchronize()
    clocks = sampler.stop(t_from, time.perf_counter())
    e2e_ms = _timed_single(lambda: ix.batch_search(q_host, k, cdb.SearchMode.HNSW, ef_search=args.ef, shortlist_size=64),
                           args.steps, 1, stream)
    ids = d_ids.cpu().numpy().view(np.uint32)
    sc = d_scores.cpu().numpy()
    # recall@10 against the exact top-10: the exact scan over the same raw rows (itself oracle-verified); the root row
    # (id = rows) is not a data row and is ignored
    gt, gts, _, _ = ix.batch_search(q_host, k + 1, cdb.SearchMode.BRUTE_RAW)
    gt = [[i for i in row if i != rows][:k] for row in gt]
    recall = float(np.mean([len(set(ids[i]) & set(gt[i])) / k for i in range(B)]))
    kernel_ms = float(np.mean(scan_ms))
    alg_bytes = evals * (D * 2 + 4) + pops * 64 * 4
    pk = _peaks()
    hbm = float(pk.get("hbm_gbs", H100_HBM_GBS))
    ach = alg_bytes / (kernel_ms / 1000.0) / 1e9
    prof = None
    if args.hnsw_prof:
        ix.hnsw_profile(enable=True, read=False)
        step()
        torch.cuda.synchronize()
        pr = ix.hnsw_profile(enable=False, read=True)
        pp_ = max(pr["pops"], 1)
        prof = {"cycles_per_pop": {k_: v / pp_ for k_, v in pr.items() if k_ != "pops"}, "pops": pr["pops"],
                "kernel": "cta-per-query (round 1)" if os.environ.get("CDB_HNSW_CTA", "0") not in ("", "0") else "warp-per-query",
                "note": "clock64 sums of lane/thread 0 over all queries of one batch / pops"}
    if args.dump_ids:
        np.savez(args.dump_ids, ids=ids, scores=sc)
    variants = None
    if args.hnsw_variants:
        # same graph, same queries: kernel time (CUDA events around the search kernel) and phase profile of every variant
        variants = []
        ref_ids = ids.copy()
        for name, fl, nb_ in [("default(preload+atomfs)", 6, B), ("speculative scoring (preload+atomfs)", 38, B), ("pool+argmax pops (preload+atomfs)", 22, B), ("preload only", 2, B),
                              ("atomfs only", 4, B), ("plain", 0, B), ("cta-per-query (round 1)", 8, B),
                              ("default, half batch", 6, B // 2), ("default, quarter batch", 6, B // 4)]:
            cdb.debug_set_hnsw_flags(fl)

            def vstep():
                ix.batch_search_device(d_q.data_ptr(), nb_, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                                       stream.cuda_stream, mode=cdb.SearchMode.HNSW, ef_search=args.ef, shortlist_size=64)
            for _ in range(2):
                vstep()
            torch.cuda.synchronize()
            for _ in range(5):
                vstep()
            torch.cuda.synchronize()
            kms = float(np.mean(ix.scan_ms_history(5)))
            same = bool(np.array_equal(d_ids.cpu().numpy().view(np.uint32)[:nb_], ref_ids[:nb_]))
            ix.hnsw_profile(enable=True, read=False)
            vstep()
            torch.cuda.synchronize()
            pr = ix.hnsw_profile(enable=False, read=True)
            pp_ = max(pr["pops"], 1)
            variants.append({"variant": name, "flags": fl, "batch": nb_, "kernel_ms": kms, "kernel_qps": nb_ / (kms / 1000.0),
                             "ids_equal_default": same, "cycles_per_pop": {k_: round(v / pp_, 2 if v < 20 * pp_ else None) for k_, v in pr.items() if k_ != "pops"}})
        cdb.debug_set_hnsw_flags()
    line = {
        "hnsw_variants": variants,
        "metric": "queries/sec + recall@10, HNSW f16", "value": args.steps * B / (ms / 1000.0), "unit": "queries/s", "n_gpus": 1,
        "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": f"{args.storage} (f32 accumulate, reference order)", "data": "synthetic (4096 Gaussian clusters)",
        "hnsw_phase_profile": prof,
        "config": {"workload": f"HNSW dense index, {rows}x{D} {args.storage}, ef_search={args.ef}, batch={B} (BASELINE.json configs[2]); graph built on the GPU "
                               "with the reference defaults", "rows": rows, "dim": D, "batch": B, "k": k},
        "clocks": clocks, "gpu_launches": int(launches),
        "e2e": {"value": args.steps * B / (e2e_ms / 1000.0), "unit": "queries/s", "h2d_bytes_per_step": B * D * 4,
                "d2h_bytes_per_step": B * k * 8 + B * 5, "ms_per_step": e2e_ms / args.steps},
        "roofline": {"bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm, "traffic": None,
                     "kernel": "hnsw_search_kernel (random row gathers)", "kernel_ms": kernel_ms, "alg_bytes_per_launch": alg_bytes,
                     "evals_per_query": evals / B, "pops_per_query": pops / B},
        "recall_at_10": recall, "build_seconds": t_build, "build_rows_per_s": rows / t_build, "load_seconds": t_load,
        "mean_top1_score": float(sc[:, 0].mean()),
    }
    print(json.dumps(line), flush=True)
    ix.close()


def run_c5(args, rank, world, local_rank):
    """BASELINE.json configs[4]: sharded HNSW, 100M x 768 fp32, batch 4096, 8 GPUs with an NCCL top-k merge.
    One independent HNSW per shard (12.5M rows per GPU by default), built on the GPU; every rank searches the same
    queries on its shard; one all-gather of the per-shard top-k; merge with the common ordering rule."""
    import torch
    import torch.distributed as dist
    import cosdata_b200 as cdb
    from cosdata_b200.sharding import ShardGroup
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    rows_local = (args.rows // world) if args.rows != 10_000_000 else 12_500_000
    rows_total = rows_local * world
    D, k = args.dim, args.k
    B = args.batch if args.batch != 1024 else 4096
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    gc = torch.Generator(device=dev)
    gc.manual_seed(1234)                                  # same centres and queries on every rank
    ncent = 4096
    centres = torch.randn((ncent, D), generator=gc, device=dev)
    scale = 1.0 / (4.5 * 1.06)
    idx = torch.randint(0, ncent, (B,), generator=gc, device=dev)
    d_q = ((centres[idx] + 0.35 * torch.randn((B, D), generator=gc, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
    g = torch.Generator(device=dev)
    g.manual_seed(777 + rank)                             # different rows per shard
    ix = cdb.DenseIndex(dim=D, storage_type=cdb.StorageType.FullPrecisionFP, metric=cdb.DistanceMetricKind.Cosine,
                        capacity=rows_local + 1, device=local_rank, id_base=rank * (rows_local + 1), tensor_prefilter=False)
    chunk = 500_000
    for off in range(0, rows_local, chunk):
        m = min(chunk, rows_local - off)
        ii = torch.randint(0, ncent, (m,), generator=g, device=dev)
        x = ((centres[ii] + 0.35 * torch.randn((m, D), generator=g, device=dev)) * scale).clamp_(-0.999, 0.999).contiguous()
        torch.cuda.synchronize()
        ix.append_device(x.data_ptr(), m)
        del x, ii
    t0 = time.perf_counter()
    ix.build_graph(9, 32, 64, 128, 64, 4096, 7 + rank)
    torch.cuda.synchronize()
    t_build = time.perf_counter() - t0
    d_ids = torch.empty((B, k), dtype=torch.int32, device=dev)
    d_scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_counts = torch.empty((B,), dtype=torch.int32, device=dev)
    # the shard group behind the C ABI owns the NCCL communicator, the gather buffer and the merge (csrc/shard_group.cu):
    # local HNSW search -> ONE ncclAllGather of packed keys -> merge, enqueued by one C call
    group = None
    if world > 1:
        box = [ShardGroup.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        group = ShardGroup.rank(box[0], world, rank, local_rank)
        group.attach(0, ix)

    def step(mode=cdb.SearchMode.HNSW):
        if group is None:
            ix.batch_search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                                   stream.cuda_stream, mode=mode, ef_search=args.ef, shortlist_size=64)
        else:
            group.search_device(d_q.data_ptr(), B, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), None,
                                stream.cuda_stream, mode=mode, ef_search=args.ef, shortlist_size=64)
        return d_ids, d_scores

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    ev0, pp0 = ix.hnsw_counters()
    for _ in range(max(args.warmup, 3)):
        step()
    barrier()
    ev1, pp1 = ix.hnsw_counters()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    l0 = cdb.kernel_launch_count()
    e0.record(stream)
    for _ in range(args.steps):
        m_ids, m_scores = step()
    e1.record(stream)
    barrier()
    if rank == 0:
        dump_device_results(args, d_ids, d_scores, d_counts)
    clocks = sampler.stop()
    launches = cdb.kernel_launch_count() - l0
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    ann = m_ids.cpu().numpy().view(np.uint32).copy()
    scan_ms = ix.scan_ms_history(args.steps * ((B + 2047) // 2048))   # before the exact scan below enters the history
    # exact global top-k for recall: exact scan of every shard (root rows excluded), same merge
    d_ids2 = torch.empty((B, k + 1), dtype=torch.int32, device=dev)
    d_sc2 = torch.empty((B, k + 1), dtype=torch.float32, device=dev)
    d_cn2 = torch.empty((B,), dtype=torch.int32, device=dev)
    ix.batch_search_device(d_q.data_ptr(), B, k + 1, d_ids2.data_ptr(), d_sc2.data_ptr(), d_cn2.data_ptr(), None,
                           stream.cuda_stream, mode=cdb.SearchMode.BRUTE_RAW)
    g2i = torch.empty((world, B, k + 1), dtype=torch.int32, device=dev)
    g2s = torch.empty((world, B, k + 1), dtype=torch.float32, device=dev)
    if world > 1:
        dist.all_gather_into_tensor(g2i.view(-1), d_ids2.view(-1))
        dist.all_gather_into_tensor(g2s.view(-1), d_sc2.view(-1))
    else:
        g2i[0], g2s[0] = d_ids2, d_sc2
    torch.cuda.synchronize()
    gi, gs = g2i.cpu().numpy().view(np.uint32), g2s.cpu().numpy()
    roots = {r * (rows_local + 1) + rows_local for r in range(world)}
    recall = 0.0
    for q in range(B):
        cand = [(float(gs[w, q, j]), int(gi[w, q, j])) for w in range(world) for j in range(k + 1) if int(gi[w, q, j]) not in roots]
        cand.sort(key=lambda t: (-t[0], t[1]))
        gt = {i for _, i in cand[:k]}
        recall += len(gt & set(ann[q].tolist())) / k
    recall /= B
    evals, pops = (ev1 - ev0) / max(args.warmup, 3), (pp1 - pp0) / max(args.warmup, 3)
    kernel_ms = float(np.sum(scan_ms)) / args.steps
    alg_bytes = evals * (D * 4 + 4) + pops * 64 * 4
    hbm = float(_peaks().get("hbm_gbs", H100_HBM_GBS))
    ach = alg_bytes / (kernel_ms / 1000.0) / 1e9
    tb = torch.tensor([t_build], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(tb, op=dist.ReduceOp.MAX)
    if rank == 0:
        line = {
            "metric": "queries/sec + recall@10, sharded HNSW f32", "value": args.steps * B / (ms / 1000.0), "unit": "queries/s",
            "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic (4096 Gaussian clusters)",
            "config": {"workload": f"sharded HNSW, {rows_total}x{D} fp32 in {world} shards of {rows_local}, ef_search={args.ef}, batch={B}, "
                                   "NCCL all-gather + top-k merge (BASELINE.json configs[4])", "rows": rows_total, "dim": D, "batch": B, "k": k},
            "clocks": clocks, "gpu_launches": int(launches),
            "roofline": {"bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm, "traffic": None,
                         "kernel": "hnsw_search_kernel (rank 0)", "kernel_ms": kernel_ms, "alg_bytes_per_launch": alg_bytes,
                         "evals_per_query": evals / B, "pops_per_query": pops / B},
            "recall_at_10": recall, "build_seconds_max_over_ranks": float(tb.item()),
        }
        print(json.dumps(line), flush=True)
    if group is not None:
        group.close()
    ix.close()
    if world > 1:
        dist.destroy_process_group()


def _watchdog(limit_s):
    """a collective that never completes must not hang the whole run: give up loudly after limit_s"""
    def bark():
        sys.stderr.write(f"bench.py: no result after {limit_s} s -- giving up (a stuck collective or kernel)\n")
        sys.stderr.flush()
        os._exit(4)
    t = threading.Timer(limit_s, bark)
    t.daemon = True
    t.start()


def main():
    args = parse_args()
    _watchdog(float(os.environ.get("CDB_BENCH_WATCHDOG_S", "1500")))
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.workload == "c5":
        run_c5(args, rank, world, local_rank)
        return
    if args.workload != "c2":
        if world != 1:
            raise SystemExit("bench.py: --workload c4/hnsw are single-GPU reporting modes")
        {"c4": run_c4, "hnsw": run_hnsw, "c3": run_c3}[args.workload](args)
        return
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    run_ours(args, rank, world, local_rank)


if __name__ == "__main__":
    main()
