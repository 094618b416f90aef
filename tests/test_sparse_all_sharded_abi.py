"""CPU-side checks of the sharded top_k None sparse search (cdb_sparse_search_batch_all_sharded): the refusals that come
before the group is read, on a stand-in group pointing at zeroed memory; the numpy merge of the ranks' variable-length
runs against a whole-corpus search by the C oracle, on shards searched one by one with their id_base; and the key
exchange's sub-batches as a function of the gathered counts alone."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import ShardGroup, key_batches, merge_runs_var, order_key_np, sparse_keys, unpack_keys
from tests import pysparse as ps
from tests import sparse_all_plan as sap
from tests.sparse_data import quirky_rows, slice_csr
from tests.text_plan import GROUP_GATHER_BUDGET

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INV = cdb.Status.INVALID_PARAMS


def last_error():
    return (_lib.load().cdb_last_error_string() or b"").decode()


def test_refusals_before_the_group_is_read():
    L = _lib.load()
    blob = (C.c_uint8 * 4096)()
    group = C.cast(blob, C.c_void_p)
    off = np.array([0, 1], np.uint64)
    dims = np.array([1], np.uint32)
    vals = np.array([1.0], np.float32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    p = cdb.SparseSearchOptions(None).params()
    out = C.c_void_p(1)

    def call(g=group, o=off, d=dims, v=vals, nq=1, params=p, res=True):
        return L.cdb_sparse_search_batch_all_sharded(g, ptr(o) if o is not None else None, ptr(d) if d is not None else None,
                                                     ptr(v) if v is not None else None, nq, C.byref(params) if params else None,
                                                     C.byref(out) if res else None)

    assert call(g=None) == INV and "null argument" in last_error()
    assert call(params=None) == INV and "null argument" in last_error()
    assert call(res=False) == INV and "null argument" in last_error()
    out.value = 1
    assert call(params=cdb.SparseSearchOptions(10).params()) == INV and "k = 0" in last_error()
    assert out.value is None                                         # *out is cleared on a refusal
    assert call(g=None, params=cdb.SparseSearchOptions(10).params()) == INV and "null argument" in last_error()   # null first
    for bad in (np.array([1, 1], np.uint64), np.array([0, 2, 1], np.uint64)):
        assert call(o=bad, nq=len(bad) - 1) == INV and "q_offsets" in last_error()
    assert call(o=None) == INV and "null offsets" in last_error()
    assert call(d=None) == INV and "null query pairs" in last_error()
    assert call(v=None) == INV and "null query pairs" in last_error()


def test_numpy_run_merge_equals_the_whole_corpus_search():
    """every shard searched alone by the oracle (k = its rows, factor 1, its id_base), its sorted keys merged by
    merge_runs_var: the whole corpus's top_k None result, with and without re-rank, deletes included"""
    rows = quirky_rows(5, 900, 30)
    rows[3] = []
    rows[4] = [(2, 0.0)]
    corpus = cdb.sparse_csr(rows)
    n = len(corpus[0]) - 1
    bounds = [0, 120, 120, 700, n]                       # an empty shard, uneven sizes
    queries = cdb.sparse_csr(quirky_rows(6, 20, 34) + [[], [(33, 1.0)]])
    deleted = np.zeros(n, np.uint8)
    deleted[np.arange(1, n, 17)] = 1
    deleted[120:130] = 1
    for bits, thr, rerank in ((4, 0.0, False), (8, 0.0, True), (6, 0.5, True), (4, float("nan"), False), (5, -0.3, True)):
        w_ids, w_scores, w_counts = ps.search(corpus, queries, n, bits=bits, thr=thr, rerank=rerank, factor=1, deleted=deleted)
        keys, counts = [], []
        for r in range(len(bounds) - 1):
            b0, b1 = bounds[r], bounds[r + 1]
            if b1 == b0:
                keys.append(np.zeros(0, np.uint64))
                counts.append(np.zeros(len(w_counts), np.int64))
                continue
            ids, scores, cnt = ps.search(slice_csr(corpus, b0, b1), queries, b1 - b0, bits=bits, thr=thr, rerank=rerank, factor=1,
                                         id_base=b0, deleted=deleted[b0:b1])
            run = []
            for q in range(len(cnt)):
                c = int(cnt[q])
                if rerank:
                    dp = scores[q, :c]
                    bits_ = np.where(np.isnan(dp), np.uint32(0xFFC00000), dp.view(np.uint32)).astype(np.uint32)
                    run.append((order_key_np(0, bits_).astype(np.uint64) << np.uint64(32)) | (~ids[q, :c]).astype(np.uint64))
                else:
                    run.append(sparse_keys(ids[q, :c], scores[q, :c].astype(np.uint64)))
            keys.append(np.concatenate(run) if run else np.zeros(0, np.uint64))
            counts.append(cnt.astype(np.int64))
        off, merged = merge_runs_var(keys, np.stack(counts))
        assert np.array_equal(np.diff(off.astype(np.int64)), w_counts.astype(np.int64))
        if rerank:
            m_ids, m_scores = unpack_keys(merged)
        else:
            m_ids = (~(merged & np.uint64(0xFFFFFFFF)).astype(np.uint32)).astype(np.uint32)
            m_scores = (merged >> np.uint64(32)).astype(np.float64).astype(np.float32)
        for q in range(len(w_counts)):
            b, e = int(off[q]), int(off[q + 1])
            assert np.array_equal(m_ids[b:e], w_ids[q, :e - b])
            assert np.array_equal(m_scores[b:e].view(np.uint32), w_scores[q, :e - b].view(np.uint32))


def test_key_batches_depend_on_the_counts_alone():
    rng = np.random.default_rng(3)
    world, c = 3, 200
    cap = GROUP_GATHER_BUDGET // (8 * world)
    counts = rng.integers(0, cap // 40, (world, c))
    counts[:, 50:60] = 0                                     # queries without a candidate anywhere
    counts[1, 100] = cap + 5                                 # one query above the budget gets a sub-batch of its own
    counts[:, 199] = 0
    got = key_batches(counts)
    assert got == key_batches(counts.copy())                 # every rank holds the same counts: the same plan
    covered = []
    for a, b, words in got:
        tot = counts[:, a:b].sum(axis=1)
        assert words == tot.max() > 0
        assert world * words * 8 <= GROUP_GATHER_BUDGET or b - a == 1
        if b < c:                                            # greedy: one more query would not fit
            assert world * (tot + counts[:, b]).max() * 8 > GROUP_GATHER_BUDGET or not (tot + counts[:, b]).any()
        covered += list(range(a, b))
    assert (100, 101, cap + 5) in got
    assert len(got) >= 3
    missing = sorted(set(range(c)) - set(covered))
    assert all(not counts[:, q].any() for q in missing)
    assert key_batches(np.zeros((2, 5), np.int64)) == []
    assert key_batches(np.array([[3, 0], [0, 4]])) == [(0, 2, 4)]


def test_budget_constant_matches_the_source():
    with open(os.path.join(ROOT, "cosdata_b200", "csrc", "sparse.cu")) as f:
        m = re.search(r"constexpr size_t SP_ALL_BUDGET = (\d+)ull << (\d+);", f.read())
    assert m and int(m.group(1)) << int(m.group(2)) == sap.SP_ALL_BUDGET


def test_scoring_chunk_plan():
    assert sap.all_chunk(10, 1, 10) == 10
    assert sap.all_chunk(100_000, 1, 1) == (512 << 20) // (32768 * 8 + 8 + 24)
    assert sap.all_chunk(100_000, 0, 0) == 65535
    assert sap.all_chunk(5000, 1, 32768) == 511
    assert sap.all_chunk(3, 700, 22_000_000) == 1                 # a query larger than the budget still runs, alone
    counts = np.zeros((2, 4), np.int64)
    assert sap.group_plan(counts, [(0, 0), (0, 0)]) == ([], [])
    assert sap.group_plan(counts, [(1, 0), (0, 0)]) == ([], [])


def test_no_cpu_fallback_without_device():
    if cdb.device_count() > 0:
        pytest.skip("CUDA device present")
    with pytest.raises(cdb.CosdataError):
        ShardGroup.local([0, 0])
