"""Sharded search behind the C ABI (csrc/shard_group.cu): the merged top-k over the shards must equal the top-k of one
index over the whole corpus -- ids and score bits -- in every mode, and the packed-key merge must follow the common
ordering rule.  One GPU: the shards share device 0 and the gather is the copy-based loopback (everything else is the
production path); with >= 2 GPUs the same checks run over a real NCCL communicator.  No torch anywhere in this file."""
import os
import subprocess

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from cosdata_b200.sharding import ShardGroup, merge_packed, pack_keys, shard_range

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def devices(n):
    return list(range(n)) if cdb.device_count() >= n else [0] * n


def make_group(corpus, nshards, **index_kw):
    n, dim = corpus.shape
    devs = devices(nshards)
    g = ShardGroup.local(devs)
    parts = []
    for r in range(nshards):
        row0, cnt = shard_range(n, nshards, r)
        ix = cdb.DenseIndex(dim=dim, capacity=cnt, device=devs[r], id_base=row0, **index_kw)
        ix.append(corpus[row0:row0 + cnt])
        g.attach(r, ix)
        parts.append(ix)
    return g, parts


@pytest.mark.parametrize("nshards,n,nq", [(2, 40000, 33), (3, 60000, 130), (2, 3000, 5)])
def test_sharded_brute_raw_equals_single_index(nshards, n, nq):
    dim, k = 128, 10
    corpus = orc.synth_matrix(5100 + nshards, n, dim)
    q = orc.synth_matrix(5200, nq, dim)
    g, parts = make_group(corpus, nshards)
    assert g.world == nshards
    ids, scores, counts, err = g.search(q, k)
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, k)
    assert np.array_equal(ids, want_ids) and np.array_equal(bits(scores), bits(want_scores))
    assert (counts == k).all() and not err.any()
    if n >= 2 * 16384:
        assert all(p.stats()["tensor_searches"] == 1 for p in parts)      # the tensor-core path ran on every shard
    ids2, scores2, _, _ = g.search(q, k, exact_only=True)
    assert np.array_equal(ids2, ids) and np.array_equal(bits(scores2), bits(scores))
    g.close()
    for p in parts:
        p.close()


def test_sharded_quantized_codes_and_error_flags():
    n, dim, nq, k = 50000, 64, 40, 7
    corpus = orc.synth_matrix(5300, n, dim).copy()
    corpus[[7, 30000]] = -1.0                     # quantize to all-zero u8 codes -> |row| = 0: cosine over codes flags every query (cosine.rs:230-231)
    q = orc.synth_matrix(5301, nq, dim)
    kw = dict(storage_type=cdb.StorageType.UnsignedByte, metric=cdb.DistanceMetricKind.Cosine)
    g, parts = make_group(corpus, 2, **kw)
    ids, scores, counts, err = g.search(q, k, cdb.SearchMode.BRUTE_CODES)
    whole = cdb.DenseIndex(dim=dim, capacity=n, **kw)
    whole.append(corpus)
    w_ids, w_scores, w_counts, w_err = whole.batch_search(q, k, cdb.SearchMode.BRUTE_CODES)
    assert np.array_equal(ids, w_ids) and np.array_equal(bits(scores), bits(w_scores))
    assert np.array_equal(err, w_err) and err.all()
    g.close(); whole.close()
    for p in parts:
        p.close()


def test_short_shards_pad_with_empty_keys():
    dim, k = 32, 10
    corpus = orc.synth_matrix(5400, 13, dim)      # shards of 5 / 4 / 4 rows < k
    q = orc.synth_matrix(5401, 6, dim)
    g, parts = make_group(corpus, 3)
    ids, scores, counts, err = g.search(q, k)
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, 13)
    assert (counts == 10).all()
    assert np.array_equal(ids, want_ids[:, :10]) and np.array_equal(bits(scores), bits(want_scores[:, :10]))
    g.close()
    for p in parts:
        p.close()


def test_sharded_hnsw_is_the_merge_of_the_per_shard_searches():
    n, dim, nq, k = 6000, 48, 24, 10
    rng = np.random.default_rng(3)
    centres = rng.normal(size=(16, dim)).astype(np.float32)
    vecs = (centres[rng.integers(0, 16, n)] + 0.3 * rng.normal(size=(n, dim))).astype(np.float32)
    vecs = (vecs / (np.abs(vecs).max() * 1.01)).astype(np.float32)
    q = (vecs[rng.integers(0, n, nq)] + 0.05 * rng.normal(size=(nq, dim))).astype(np.float32)
    devs = devices(2)
    g = ShardGroup.local(devs)
    parts, per = [], []
    for r in range(2):
        row0, cnt = shard_range(n, 2, r)
        ix = cdb.DenseIndex(dim=dim, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=cnt + 1, device=devs[r],
                            id_base=r * (n // 2 + 1), keep_raw_f32=True)
        ix.append(vecs[row0:row0 + cnt])
        ix.build_graph(4, 8, 16, 64, 64, 1, 11 + r)          # one vector at a time: deterministic graph
        g.attach(r, ix)
        parts.append(ix)
        per.append(ix.batch_search(q, k, cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64))
    ids, scores, counts, err = g.search(q, k, cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64)
    gathered = np.stack([pack_keys(p[0], p[1]) for p in per])
    w_ids, w_scores, w_counts = merge_packed(gathered, k)
    assert np.array_equal(ids, w_ids) and np.array_equal(bits(scores), bits(w_scores)) and np.array_equal(counts, w_counts)
    g.close()
    for p in parts:
        p.close()


def test_rank_group_of_one_needs_no_nccl():
    corpus = orc.synth_matrix(5500, 20000, 64)
    q = orc.synth_matrix(5501, 9, 64)
    g = ShardGroup.rank(None, 1, 0, 0)
    ix = cdb.DenseIndex(dim=64, capacity=20000)
    ix.append(corpus)
    g.attach(0, ix)
    ids, scores, _, _ = g.search(q, 10)
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, 10)
    assert np.array_equal(ids, want_ids) and np.array_equal(bits(scores), bits(want_scores))
    g.close(); ix.close()


@pytest.mark.parametrize("ndev", [0, 2])
def test_plain_c_host_program_runs_the_sharded_search(tmp_path, ndev):
    """tests/cpp/shard_smoke.cpp: C ABI only (what a Rust host binds); ndev = 2 uses NCCL when two GPUs are present"""
    exe = str(tmp_path / "shard_smoke")
    libdir = os.path.join(ROOT, "cosdata_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "shard_smoke.cpp"), "-o", exe, "-L", libdir, "-lcosdata_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([exe, str(ndev)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "merged_equals_whole=1" in r.stdout or "skipped" in r.stdout, r.stdout
