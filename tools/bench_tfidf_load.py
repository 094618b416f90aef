"""TF-IDF restart from the reference's files: a 1M-document Zipf corpus (tests/tfidf_data.zipf_docs) written once as the
reference's tf_idf_index files -- two versions, 1 % of the documents deleted in the second -- then timed, median of
--steps runs after one warm-up:
  open        cdb_tfidf_files_open (tree walk, chains, tombstones; the host reads the files)
  load        cdb_tfidf_index_load_files into a new index: wall time; CUDA events on the caller's stream around the call
              (the device-side span: the load drains the device first and returns with its work finished, so the span
              covers its device work and the host staging between it); and, in 5 further loads, the device's busy time
              inside the call (kernels and copies, from torch.profiler)
  host path   for comparison: cdb_tfidf_files_read, a numpy transposition of the live postings into row CSR, and
              cdb_tfidf_index_append of those rows (what a shim without the device load would do; it cannot restore the
              files' df and N, so only its time is compared)
Parity: a 64-query batch on the loaded index and on an index fed the same appends and deletes must give identical ids,
counts and score bits at k = 10 and k = 0.  Prints the card and its power limit, then one JSON line.

    python tools/bench_tfidf_load.py [--rows 1000000] [--steps 5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosdata_b200 as cdb  # noqa: E402
from tests import tfidf_files as tff  # noqa: E402
from tests.tfidf_data import zipf_docs, zipf_queries  # noqa: E402

VOCAB = 1_000_000


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def device_busy_ms(fn):
    """fn() under torch.profiler -> summed device time of its kernels and copies (ms), or None"""
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            fn()
        return sum(e.device_time_total for e in p.events() if e.device_time_total) / 1e3
    except Exception:
        return None


def host_path(files, n, n1, cap_pairs):
    hs, df, off, ids, tfs, ver = files.read()
    h = np.repeat(hs, np.diff(off).astype(np.int64))
    order = np.argsort(ids, kind="stable")
    counts = np.bincount(ids, minlength=n)
    roff = np.zeros(n + 1, np.uint64)
    roff[1:] = np.cumsum(counts)
    rh, rt = h[order], tfs[order]
    ix = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=cap_pairs)
    p1 = int(roff[n1])
    ix.append((roff[:n1 + 1], rh[:p1], rt[:p1]), 1)
    ix.append((roff[n1:] - roff[n1], rh[p1:], rt[p1:]), 2)
    return ix


def median(xs):
    return float(np.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    import torch
    assert cdb.device_count() > 0, "needs a CUDA device"
    print(json.dumps({"card": card()}), flush=True)
    n = a.rows
    off, hs, tf = zipf_docs(1000, n, vocab=VOCAB)
    n1 = n // 2
    dele = np.sort(np.random.default_rng(5).choice(n1, n // 100, replace=False))
    mask = np.ones(n, np.uint8)
    mask[dele] = 0
    tmp = tempfile.mkdtemp(prefix="cdb_tfidf_load_")
    try:
        d = os.path.join(tmp, "tf_idf_index")
        t0 = time.perf_counter()
        tff.write_bulk(d, off, hs, tf, n1, dele)
        write_s = time.perf_counter() - t0
        cap = len(hs) + 64
        # the same history fed to the GPU index
        ref = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=cap)
        p1 = int(off[n1])
        ref.append((off[:n1 + 1], hs[:p1], tf[:p1]), 1)
        ref.append((off[n1:] - off[n1], hs[p1:], tf[p1:]), 2)
        ref.delete_embedding(dele, 2)
        t_open, t_load, t_host, t_event, busy = [], [], [], [], []
        for step in range(a.steps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f = cdb.TfIdfFiles(d)
            t1 = time.perf_counter()
            ix = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=cap)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t2 = time.perf_counter()
            e0.record()
            ix.load_files(f, n, counted=mask)
            e1.record()
            t3 = time.perf_counter()
            e1.synchronize()
            hx_t0 = time.perf_counter()
            hx = host_path(f, n, n1, cap)
            hx_t1 = time.perf_counter()
            if step:
                t_open.append(t1 - t0)
                t_load.append(t3 - t2)
                t_host.append(hx_t1 - hx_t0)
                t_event.append(e0.elapsed_time(e1))
            if step == a.steps:
                for _ in range(a.steps):
                    ix2 = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=cap)
                    busy.append(device_busy_ms(lambda: ix2.load_files(f, n, counted=mask)))
                    ix2.close()
            info = f.info
            f.close()
            hx.close()
            if step < a.steps:
                ix.close()
        qs = zipf_queries(7, 64, vocab=VOCAB)
        parity = True
        for k in (10, 0):
            i1, s1, c1 = ix.batch_search(qs, k)
            i2, s2, c2 = ref.batch_search(qs, k)
            parity &= bool(np.array_equal(i1, i2) and np.array_equal(c1, c2) and np.array_equal(s1.view(np.uint32), s2.view(np.uint32)))
        df1, idf1, n_1 = ix.term_stats(np.unique(hs)[::97])
        df2, idf2, n_2 = ref.term_stats(np.unique(hs)[::97])
        parity &= bool(n_1 == n_2 and np.array_equal(df1, df2) and np.array_equal(idf1.view(np.uint32), idf2.view(np.uint32)))
        ix.close()
        ref.close()
        out = {"rows": n, "pairs": int(len(hs)), "live_words": info["live"], "records": info["records"], "terms": info["terms"],
               "write_files_s": round(write_s, 2), "open_ms": round(1e3 * median(t_open), 1), "load_ms": round(1e3 * median(t_load), 1),
               "load_event_span_ms": round(median(t_event), 1),
               "load_device_busy_ms": None if None in busy else round(median(busy), 1),
               "host_read_transpose_append_ms": round(1e3 * median(t_host), 1), "parity": parity, "steps": a.steps}
        print(json.dumps(out), flush=True)
        if not parity:
            sys.exit(1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
