"""Sparse search with top_k None (cdb_sparse_search_batch_all): every candidate of every query, scored, optionally re-ranked
and sorted on the GPU, against the CPU oracle (tests/sparse_oracle.c) run with k = n_rows and factor 1, which cuts nothing
and re-ranks every candidate.  Counts, ids and score bits are compared exactly: on the reference's quirks (bits 4-8, every
early-termination threshold, zero / negative / NaN values, duplicate dims, rows reached only by zero products, empty rows
and queries, absent dims), on corpora of several row tiles appended in pieces with deletes, across query chunks, and at
1M rows.  Also: agreement with the top-k search, the result handle's reads, offsets, independence from the index and
refusals, and searches from 8 host threads."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from tests import pysparse as ps
from tests.sparse_data import concat_csr, quirky_rows, slice_csr, zipf_csr

pytestmark = pytest.mark.gpu

THRS = [0.0, 0.5, 1.0, 1.7, -0.3, float("nan")]


def opts_all(thr=0.0, rerank=False, factor=5):
    return cdb.SparseSearchOptions(None, thr, rerank, factor)


def oracle_all(corpus, queries, thr=0.0, rerank=False, bits=4, ub=1.0, deleted=None, id_base=0):
    """top_k None in the oracle: k = n_rows, factor 1"""
    n = len(corpus[0]) - 1
    return ps.search(corpus, queries, max(n, 1), bits=bits, ub=ub, thr=thr, rerank=rerank, factor=1, id_base=id_base,
                     deleted=deleted)


def check_all(got, want, sample=None):
    """got: (offsets, ids, scores) of the whole batch; want: the oracle's (ids, scores, counts) of the queries in sample"""
    off, ids, scores = got
    w_ids, w_scores, w_counts = want
    counts = np.diff(off.astype(np.int64))
    qs = np.arange(len(counts)) if sample is None else np.asarray(sample)
    assert np.array_equal(counts[qs], w_counts.astype(np.int64))
    for i, q in enumerate(qs):
        b, e, c = int(off[q]), int(off[q + 1]), int(w_counts[i])
        assert np.array_equal(ids[b:e], w_ids[i, :c]), q
        assert np.array_equal(scores[b:e].view(np.uint32), w_scores[i, :c].view(np.uint32)), q


def same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))


def sample_csr(queries, sample):
    return concat_csr([slice_csr(queries, int(i), int(i) + 1) for i in sample])


@pytest.mark.parametrize("bits", [4, 5, 6, 7, 8])
def test_quirks_against_the_oracle(bits):
    rows = quirky_rows(1 + bits, 3000, 40)
    rows[5] = [(7, 0.0)]                        # touched only through zero products
    rows[6] = []                                # empty row: never a candidate
    rows[7] = [(3, 0.2), (3, 0.9), (3, 0.4)]    # duplicate dims: counted thrice, the last wins the re-rank
    corpus = cdb.sparse_csr(rows)
    ub = 1.5 if bits % 2 else 1.0
    ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=4000, capacity_pairs=len(corpus[1]) + 10,
                         id_base=17)
    ix.append(corpus)
    queries = quirky_rows(100 + bits, 60, 45)   # dims 40..44 are absent from the index
    queries[0] = []
    queries[1] = [(7, 0.0)]
    queries[2] = [(3, 0.5), (3, 0.5), (9, 2.0)]
    queries[3] = [(41, 1.0)]
    q = cdb.sparse_csr(queries)
    for thr in THRS:
        for rerank in (False, True):
            got = ix.batch_search_all(q, opts_all(thr, rerank))
            check_all(got, oracle_all(corpus, q, thr, rerank, bits, ub, id_base=17))
    off, ids, _ = ix.batch_search_all(q, opts_all(0.0))
    assert off[1] == 0                                          # the empty query
    assert 17 + 5 in ids[off[1]:off[2]].tolist()                # a row reached only by a zero product is a candidate
    assert 17 + 6 not in ids.tolist()                           # an empty row never is
    ix.close()


def test_tiles_appended_in_pieces_with_deletes():
    corpus = zipf_csr(7, 100_000, vocab=3000, mean_pairs=30)
    n = len(corpus[0]) - 1
    ix = cdb.SparseIndex(quantization_bits=6, values_upper_bound=3.0, capacity_rows=n, capacity_pairs=len(corpus[1]), id_base=1000)
    queries = zipf_csr(8, 24, vocab=3000, mean_pairs=12)
    deleted = np.zeros(n, np.uint8)
    cuts = [0, 30_001, 70_000, n]                # pieces end mid-tile (tiles hold 32768 rows)
    ix.append(slice_csr(corpus, cuts[0], cuts[1]))
    part = slice_csr(corpus, 0, cuts[1])
    check_all(ix.batch_search_all(queries, opts_all()), oracle_all(part, queries, bits=6, ub=3.0, id_base=1000))
    ix.append(slice_csr(corpus, cuts[1], cuts[2]))
    ix.append(slice_csr(corpus, cuts[2], cuts[3]))
    # the row that ranks first for query 0, with and without re-rank, is deleted along with rows in every tile
    firsts = []
    for rerank in (False, True):
        off, ids, _ = ix.batch_search_all(slice_csr(queries, 0, 1), opts_all(0.0, rerank))
        assert off[1] > 0
        firsts.append(int(ids[0]) - 1000)
    dels = np.unique(np.concatenate([np.array(firsts), np.arange(5, n, 997), [0, 32_767, 32_768, 65_536, n - 1]])).astype(np.uint32)
    ix.delete_embedding(dels)
    deleted[dels] = 1
    for thr, rerank in ((0.0, False), (0.0, True), (0.3, False), (0.3, True)):
        got = ix.batch_search_all(queries, opts_all(thr, rerank))
        check_all(got, oracle_all(corpus, queries, thr, rerank, 6, 3.0, deleted, 1000))
        assert not np.isin(got[1], dels.astype(np.uint64) + 1000).any()
    ix.close()


def test_first_results_equal_the_top_k_search():
    corpus = zipf_csr(21, 70_000, vocab=2000, mean_pairs=25)
    queries = zipf_csr(22, 40, vocab=2000, mean_pairs=10)
    queries = concat_csr([queries, cdb.sparse_csr([[], [(1999, 0.01)]])])
    ix = cdb.SparseIndex(capacity_rows=70_000, capacity_pairs=len(corpus[1]), values_upper_bound=2.0)
    ix.append(corpus)
    ix.delete_embedding(np.arange(0, 70_000, 13, dtype=np.uint32))
    for thr in (0.0, 0.5):
        off, ids, scores = ix.batch_search_all(queries, opts_all(thr))
        counts = np.diff(off.astype(np.int64))
        for k in (1, 10, 1024):
            t_ids, t_scores, t_counts = ix.batch_search(queries, cdb.SparseSearchOptions(k, thr))
            assert np.array_equal(t_counts, np.minimum(counts, k))
            for q in range(len(counts)):
                c, b = int(t_counts[q]), int(off[q])
                assert np.array_equal(ids[b:b + c], t_ids[q, :c])
                assert np.array_equal(scores[b:b + c].view(np.uint32), t_scores[q, :c].view(np.uint32))
    ix.close()


def test_chunked_batch():
    """4 row tiles and ~1100 short queries: the batch is searched in several chunks under the scratch budget"""
    corpus = zipf_csr(31, 120_000, vocab=3000, mean_pairs=20)
    queries = zipf_csr(32, 1100, vocab=3000, mean_pairs=4)
    ix = cdb.SparseIndex(quantization_bits=5, capacity_rows=120_000, capacity_pairs=len(corpus[1]), values_upper_bound=2.0,
                         id_base=5)
    ix.append(corpus)
    ix.delete_embedding(np.arange(3, 120_000, 101, dtype=np.uint32))
    deleted = np.zeros(120_000, np.uint8)
    deleted[np.arange(3, 120_000, 101)] = 1
    sample = np.arange(0, 1100, 73)
    for rerank in (False, True):
        got = ix.batch_search_all(queries, opts_all(0.0, rerank))
        check_all(got, oracle_all(corpus, sample_csr(queries, sample), 0.0, rerank, 5, 2.0, deleted, 5), sample)
        parts = [ix.batch_search_all(slice_csr(queries, a, min(a + 100, 1100)), opts_all(0.0, rerank)) for a in range(0, 1100, 100)]
        off = np.concatenate([np.zeros(1, np.uint64)] + [p[0][1:] + np.uint64(sum(int(x[0][-1]) for x in parts[:i]))
                                                          for i, p in enumerate(parts)])
        same(got, (off, np.concatenate([p[1] for p in parts]), np.concatenate([p[2] for p in parts])))
    ix.close()


def test_result_handle():
    L = _lib.load()
    corpus = zipf_csr(41, 40_000, vocab=1500, mean_pairs=20)
    queries = zipf_csr(42, 30, vocab=1500, mean_pairs=8)
    queries = concat_csr([slice_csr(queries, 0, 10), cdb.sparse_csr([[]]), slice_csr(queries, 10, 30)])
    ix = cdb.SparseIndex(capacity_rows=50_000, capacity_pairs=len(corpus[1]) + 200_000, values_upper_bound=2.0)
    ix.append(corpus)
    opts = opts_all(0.0, True, 0)                       # reranking_factor 0 is accepted (ignored) with top_k None
    r = ix.search_all_results(queries, opts)
    off = r.offsets()
    assert len(off) == 32 and off[0] == 0 and np.all(np.diff(off.astype(np.int64)) >= 0) and off[11] == off[10]
    full = r.read(0, 31)
    assert len(full[0]) == off[-1]
    check_all((off,) + full, oracle_all(corpus, queries, 0.0, True, ub=2.0))
    rng = np.random.default_rng(0)
    for _ in range(20):
        a = int(rng.integers(0, 32))
        b = int(rng.integers(a, 32))
        ids, scores = r.read(a, b - a)
        assert np.array_equal(ids, full[0][off[a]:off[b]])
        assert np.array_equal(scores.view(np.uint32), full[1][off[a]:off[b]].view(np.uint32))
    # the handle does not reference the index
    ix.append(zipf_csr(43, 5000, vocab=1500, mean_pairs=20))
    ix.delete_embedding(full[0][:50])
    assert not np.array_equal(ix.batch_search_all(queries, opts)[1], full[0])
    ix.close()
    assert np.array_equal(r.offsets(), off)
    got = r.read(0, 31)
    assert np.array_equal(got[0], full[0]) and np.array_equal(got[1].view(np.uint32), full[1].view(np.uint32))
    # refusals: read range, null pointers
    for a, n in ((0, 32), (31, 1), (32, 0), (1 << 31, 1 << 31)):
        assert L.cdb_sparse_results_read(r.h, a, n, None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_sparse_results_read(r.h, 0, 1, None, None) == (cdb.Status.OK if off[1] == 0 else cdb.Status.INVALID_PARAMS)
    assert L.cdb_sparse_results_read(None, 0, 0, None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_sparse_results_offsets(r.h, None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_sparse_results_read(r.h, 10, 1, None, None) == cdb.Status.OK     # the empty query: nothing to copy
    r.close()
    assert L.cdb_sparse_results_destroy(None) == cdb.Status.OK


def test_empty_batches_indexes_and_refusals():
    L = _lib.load()
    empty = cdb.SparseIndex(capacity_rows=10, capacity_pairs=10)
    before = cdb.kernel_launch_count()
    off, ids, scores = empty.batch_search_all([[(1, 1.0)], [], [(2, 0.5)]], opts_all(0.0, True))
    assert off.tolist() == [0, 0, 0, 0] and len(ids) == 0 and len(scores) == 0
    off, ids, _ = empty.batch_search_all([], opts_all())
    assert off.tolist() == [0] and len(ids) == 0
    assert empty.search([(1, 1.0)], opts_all()) == []
    assert cdb.kernel_launch_count() == before
    empty.close()

    ix = cdb.SparseIndex(capacity_rows=10, capacity_pairs=10, id_base=4)
    ix.append([[(1, 0.5)], [(1, 0.25), (2, 1.0)], []])
    assert ix.batch_search_all([], opts_all())[0].tolist() == [0]
    res = ix.search([(1, 1.0)], opts_all())
    assert [i for i, _ in res] == [4, 5] and res == ix.search([(1, 1.0)], cdb.SparseSearchOptions(10))
    ix.delete_embedding([0, 1])
    assert ix.batch_search_all([[(1, 1.0)]], opts_all())[0].tolist() == [0, 0]     # no live candidate left
    for o in (cdb.SparseSearchOptions(1), cdb.SparseSearchOptions(10, rerank=True)):
        with pytest.raises(cdb.CosdataError) as e:
            ix.batch_search_all([[(1, 1.0)]], o)
        assert e.value.status == cdb.Status.INVALID_PARAMS
    p = opts_all().params()
    out = C.c_void_p(1)
    qo = np.array([0, 1], np.uint64)
    qd = np.array([1], np.uint32)
    qv = np.array([1.0], np.float32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    inv = cdb.Status.INVALID_PARAMS
    assert L.cdb_sparse_search_batch_all(None, ptr(qo), ptr(qd), ptr(qv), 1, C.byref(p), C.byref(out)) == inv
    assert L.cdb_sparse_search_batch_all(ix.h, ptr(qo), ptr(qd), ptr(qv), 1, None, C.byref(out)) == inv
    assert L.cdb_sparse_search_batch_all(ix.h, ptr(qo), ptr(qd), ptr(qv), 1, C.byref(p), None) == inv
    assert L.cdb_sparse_search_batch_all(ix.h, None, ptr(qd), ptr(qv), 1, C.byref(p), C.byref(out)) == inv
    assert out.value is None                                         # *out is cleared on a refusal
    assert L.cdb_sparse_search_batch_all(ix.h, ptr(qo), None, ptr(qv), 1, C.byref(p), C.byref(out)) == inv
    for bad in (np.array([1, 1], np.uint64), np.array([0, 2, 1], np.uint64)):
        assert L.cdb_sparse_search_batch_all(ix.h, ptr(bad), ptr(qd), ptr(qv), len(bad) - 1, C.byref(p), C.byref(out)) == inv
    with pytest.raises(cdb.CosdataError) as e:                       # the top-k entry point still refuses k = 0
        ix.batch_search([[(1, 1.0)]], opts_all())
    assert e.value.status == inv
    ix.close()


def test_threads_equal_the_serial_results():
    corpus = zipf_csr(51, 40_000, vocab=2000, mean_pairs=25)
    queries = zipf_csr(52, 64, vocab=2000, mean_pairs=10)
    ix = cdb.SparseIndex(capacity_rows=40_000, capacity_pairs=len(corpus[1]), values_upper_bound=2.0)
    ix.append(corpus)
    for rerank in (False, True):
        want = ix.batch_search_all(queries, opts_all(0.0, rerank))
        with concurrent.futures.ThreadPoolExecutor(8) as ex:
            for got in ex.map(lambda _: ix.batch_search_all(queries, opts_all(0.0, rerank)), range(16)):
                same(got, want)
    r = ix.search_all_results(queries, opts_all(0.2, True))
    full = r.read(0, 64)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        for got in ex.map(lambda _: r.read(0, 64), range(16)):
            assert np.array_equal(got[0], full[0]) and np.array_equal(got[1].view(np.uint32), full[1].view(np.uint32))
    r.close()
    ix.close()


def test_one_million_rows_batch_16():
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < 8 << 30:
        pytest.skip("needs 8 GB of free device memory")
    corpus = zipf_csr(11, 1_000_000, mean_pairs=120)
    queries = zipf_csr(12, 16, mean_pairs=40)
    ix = cdb.SparseIndex(capacity_rows=1_000_000, capacity_pairs=len(corpus[1]), values_upper_bound=3.0)
    ix.append(corpus)
    sample = np.array([0, 5, 15])
    for rerank in (False, True):
        got = ix.batch_search_all(queries, opts_all(0.5, rerank))
        assert int(got[0][-1]) > 16 * 100
        check_all(got, oracle_all(corpus, sample_csr(queries, sample), 0.5, rerank, ub=3.0), sample)
    ix.close()
