"""bench.py contract (CPU side): the reference arm prints ONE JSON line with the agreed keys, runs without a GPU, and only
rank 0 works under a multi-rank launch; --dump-outputs writes the last step's results, identical from run to run."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = ["--impl", "reference", "--steps", "2", "--warmup", "1", "--cpu-sample-rows", "20000", "--cpu-sample-queries", "4"]


def run(extra_env, extra_args=()):
    env = dict(os.environ, **extra_env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + ARGS + list(extra_args), capture_output=True, text=True,
                          env=env, timeout=600)


def load_bench():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    return bench


def test_reference_arm_line():
    r = run({})
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in d, key
    assert d["impl"] == "reference" and d["steps"] == 2 and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["value"] > 0 and d["unit"] == "queries/s" and "workload" in d["config"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_other_ranks_do_nothing():
    r = run({"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2", "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": "29571"})
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == ""


def test_clock_sampling_repeats_are_a_pure_function_of_the_reduced_time():
    # the untimed repeats contain NCCL collectives: every rank must derive the same count (a time-based loop per rank hung the
    # 8-GPU run of round 2).  The count only depends on values that are identical on all ranks.
    f = load_bench().clock_sampling_repeats
    assert f(120.0, 10, 3) == 8                      # 12 ms steps: 156 ms of load so far, 94 ms missing -> 8 more steps
    assert f(16.0, 10, 3) == 144                     # 1.6 ms steps (8 GPUs): 20.8 ms so far -> 144 more
    assert f(5000.0, 10, 3) == 0                     # long steps: nothing to add
    assert f(0.0, 10, 3) == 2000 and f(1e-9, 1, 0) == 2000      # degenerate timings are capped
    assert all(f(t, 5, 3) == f(t, 5, 3) for t in (1.0, 33.3, 250.0))


def test_dump_outputs_writes_float_arrays_by_name_within_the_limit(tmp_path):
    bench = load_bench()
    ids = np.arange(40, dtype=np.float64).reshape(4, 10)
    scores = np.linspace(-1, 1, 40, dtype=np.float32).reshape(4, 10)
    bench.dump_outputs(str(tmp_path / "out"), ids=ids, scores=scores)
    assert sorted(os.listdir(tmp_path / "out")) == ["ids.npy", "scores.npy"]
    got = np.load(tmp_path / "out" / "scores.npy")
    assert got.dtype == np.float32 and np.array_equal(got, scores)
    assert np.array_equal(np.load(tmp_path / "out" / "ids.npy"), ids)
    with pytest.raises(ValueError):                                          # integer arrays are not accepted
        bench.dump_outputs(str(tmp_path / "bad"), ids=ids.astype(np.uint32))
    big = np.zeros(bench.DUMP_LIMIT_BYTES // 8 + 1, dtype=np.float64)        # one element over 64 MB
    with pytest.raises(ValueError):
        bench.dump_outputs(str(tmp_path / "big"), big=big)
    assert not (tmp_path / "bad").exists() and not (tmp_path / "big").exists()   # nothing written on refusal


def test_reference_arm_dumps_the_same_outputs_every_run(tmp_path):
    got = []
    for i in range(2):
        d = tmp_path / f"run{i}"
        r = run({}, ["--dump-outputs", str(d)])
        assert r.returncode == 0, r.stderr[-2000:]
        assert sorted(os.listdir(d)) == ["ids.npy", "scores.npy"]
        ids, scores = np.load(d / "ids.npy"), np.load(d / "scores.npy")
        assert ids.dtype == np.float64 and scores.dtype == np.float32 and ids.shape == scores.shape == (4, 10)
        assert np.all(ids == np.floor(ids)) and ids.min() >= 0 and ids.max() < 20000
        got.append((ids, scores))
    assert np.array_equal(got[0][0], got[1][0]) and np.array_equal(got[0][1].view(np.uint32), got[1][1].view(np.uint32))
