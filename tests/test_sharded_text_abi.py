"""CPU-side checks of the sharded sparse and TF-IDF search: the C ABI refuses bad calls before any device work, and the numpy
restatements of the merges in cosdata_b200/sharding.py equal the whole-corpus C oracle when each shard is searched on its
own (tests/sparse_oracle.c with id_base), including a corpus where re-ranking each shard's own top k * f and then merging
would not."""
import ctypes as C

import numpy as np

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import INVALID_ID, merge_buckets, merge_sparse, pack_keys, sparse_keys
from tests import pysparse as ps
from tests.sparse_data import slice_csr, zipf_csr


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def last_error():
    return (_lib.load().cdb_last_error_string() or b"").decode()


def test_refusals_before_touching_the_device():
    L = _lib.load()
    inv = cdb.Status.INVALID_PARAMS
    qo, qd, qv = np.array([0, 1], np.uint64), np.array([1], np.uint32), np.array([1.0], np.float32)
    ids, scores, counts = np.zeros(8, np.uint32), np.zeros(8, np.float32), np.zeros(1, np.uint32)
    args = (ptr(qo), ptr(qd), ptr(qv), 1)
    outs = (ptr(ids), ptr(scores), ptr(counts))
    for opts, msg in ((cdb.SparseSearchOptions(None), "k must be"), (cdb.SparseSearchOptions(1025), "k must be"),
                      (cdb.SparseSearchOptions(1024, rerank=True, reranking_factor=6), "reranking_factor"),
                      (cdb.SparseSearchOptions(8), "null argument")):
        p = opts.params()
        assert L.cdb_sparse_search_batch_sharded(None, *args, C.byref(p), *outs) == inv and msg in last_error()
        assert L.cdb_sparse_search_batch_sharded_device(None, *args, C.byref(p), *outs, None) == inv and msg in last_error()
    assert L.cdb_sparse_search_batch_sharded(None, *args, None, *outs) == inv
    assert L.cdb_tfidf_search_batch_sharded(None, ptr(qo), ptr(qd), 1, 10, *outs) == inv and "null argument" in last_error()
    assert L.cdb_shard_group_attach_sparse(None, 0, None) == inv
    assert L.cdb_shard_group_attach_tfidf(None, 0, None) == inv


def rerank_fn(corpus, queries):
    """finalize_sparse_ann_results' dot product in f32, one rounding per operation, query pairs in the caller's order"""
    (ro, rd, rv), (qo, qd, qv) = corpus, queries

    def fn(q, ids):
        out = np.zeros(len(ids), np.float32)
        for i, gid in enumerate(ids):
            a, b = int(ro[gid]), int(ro[gid + 1])
            row = dict(zip(rd[a:b].tolist(), rv[a:b]))          # a row's last pair of a dim wins
            dp = np.float32(0.0)
            for d, v in zip(qd[int(qo[q]):int(qo[q + 1])].tolist(), qv[int(qo[q]):int(qo[q + 1])]):
                if d in row:
                    dp = np.float32(dp + np.float32(row[d] * v))
            out[i] = dp
        return out
    return fn


def per_shard_keys(corpus, queries, bounds, m, thr=0.0):
    """every shard's top m by similarity, as the oracle finds it on that shard alone -> [world, B, m] keys"""
    keys = []
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        ids, scores, _ = ps.search(slice_csr(corpus, b0, b1), queries, m, thr=thr, id_base=b0)
        keys.append(sparse_keys(ids, scores.astype(np.uint32)))     # similarities stay below 2^24 here: exact as f32
    return np.stack(keys)


def check(got, want):
    for a, b in zip(got, want):
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_sparse_merge_mirror_equals_the_whole_corpus_oracle():
    n = 900
    corpus = zipf_csr(41, n, vocab=300, mean_pairs=10)
    queries = zipf_csr(42, 24, vocab=300, mean_pairs=5)
    for bounds in ([0, 450, n], [0, 100, 101, 700, n], [0, 0, n]):
        for thr in (0.0, 0.5):
            for k in (1, 10, 40):
                check(merge_sparse(per_shard_keys(corpus, queries, bounds, k, thr), k), ps.search(corpus, queries, k, thr=thr))
            for k, f in ((1, 5), (10, 5), (7, 3)):
                got = merge_sparse(per_shard_keys(corpus, queries, bounds, k * f, thr), k, rerank_fn(corpus, queries))
                check(got, ps.search(corpus, queries, k, thr=thr, rerank=True, factor=f))


def test_two_phase_rerank_differs_from_rerank_per_shard():
    """k = 1, f = 2.  Rows 0 and 1 (shard 0) and 10 and 11 (shard 1) have the same similarity; the group's top 2 are 0 and 1
    (ties to the smaller id), whose raw value is lower than 10's.  Re-ranking each shard's own top 2 and merging returns 10."""
    rows = [[(0, 1.0)], [(0, 1.0)]] + [[]] * 8 + [[(0, 5.0)], [(0, 5.0)]]
    corpus = cdb.sparse_csr(rows)
    queries = cdb.sparse_csr([[(0, 1.0)]])
    bounds = [0, 10, 12]
    want = ps.search(corpus, queries, 1, rerank=True, factor=2)
    assert want[0][0, 0] == 0 and want[1][0, 0] == 1.0
    check(merge_sparse(per_shard_keys(corpus, queries, bounds, 2), 1, rerank_fn(corpus, queries)), want)
    # the per-shard form: each shard re-ranks its own top 2, then the re-ranked keys are merged
    per = [ps.search(slice_csr(corpus, b0, b1), queries, 1, rerank=True, factor=2, id_base=b0) for b0, b1 in zip(bounds[:-1], bounds[1:])]
    keys = np.concatenate([pack_keys(i, s) for i, s, _ in per], axis=1)
    best = keys[0].max()
    assert (~np.uint32(best & np.uint64(0xFFFFFFFF))) == 10


def test_bucket_merge_ties_go_to_the_smaller_id():
    """rank 0 holds the larger ids: equal scores (+0 / -0 too) in one bucket go to the smaller id on rank 1"""
    g_ids = np.full((2, 1, 512), INVALID_ID, np.uint32)
    g_scores = np.full((2, 1, 512), -np.inf, np.float32)
    g_ids[0, 0, 5], g_scores[0, 0, 5] = 1029, 2.0
    g_ids[1, 0, 5], g_scores[1, 0, 5] = 5, 2.0
    g_ids[0, 0, 7], g_scores[0, 0, 7] = 1031, 0.0
    g_ids[1, 0, 7], g_scores[1, 0, 7] = 7, -0.0
    g_ids[0, 0, 9], g_scores[0, 0, 9] = 1033, 3.0
    g_ids[1, 0, 9], g_scores[1, 0, 9] = 9, 1.0
    ids, scores, counts = merge_buckets(g_ids, g_scores, 10)
    assert counts[0] == 3
    assert ids[0, :3].tolist() == [1033, 5, 7]
    assert scores[0, 2] == 0.0 and np.signbit(scores[0, 2])
    ids, _, counts = merge_buckets(g_ids, g_scores, 0)
    assert ids.shape == (1, 512) and counts[0] == 3
