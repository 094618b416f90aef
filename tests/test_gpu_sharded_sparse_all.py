"""Sharded sparse search with top_k None (cdb_sparse_search_batch_all_sharded): offsets, ids and score bits must equal what
cdb_sparse_search_batch_all returns on ONE index holding every shard's rows at their global ids, with the same appends and
deletes, with and without re-rank; a sample also against the C oracle (k = n_rows, factor 1).  Groups of 2, 3 and 4 uneven
shards, bits 4 and 8, every threshold of test_gpu_sparse_all, quirky rows, deletes on several shards, empty and all-deleted
shards, queries without a candidate, a skewed corpus, a batch of two scoring chunks whose key exchange splits, a per-rank
group of one rank, the handle's independence from the shards, and the refusals.  One GPU: the shards share device 0 and
the gathers are the copy-based loopback; with >= 2 GPUs the same checks run over a real NCCL communicator."""
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.api import SparseResults
from cosdata_b200.sharding import ShardGroup
from tests import sparse_all_plan as sap
from tests.sparse_data import concat_csr, quirky_rows, slice_csr, zipf_csr
from tests.test_gpu_sparse_all import THRS, check_all, oracle_all, opts_all, same, sample_csr

pytestmark = pytest.mark.gpu


def devices(n):
    return list(range(n)) if cdb.device_count() >= n else [0] * n


def sparse_group(corpus, bounds, bits=4, ub=1.0, room=0):
    """shards over rows [bounds[r], bounds[r+1]) of corpus (an empty range: a shard without rows); the last shard has
    capacity for `room` more rows and pairs"""
    n = len(bounds) - 1
    devs = devices(n)
    g = ShardGroup.local(devs)
    parts = []
    for r in range(n):
        b0, b1 = bounds[r], bounds[r + 1]
        base = b0 if b1 > b0 else bounds[-1] + r          # an empty shard: one row of capacity past every other range
        extra = room if r == n - 1 else 0
        ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=max(b1 - b0, 1) + extra,
                             capacity_pairs=int(corpus[0][b1] - corpus[0][b0]) + 8 + 64 * extra, id_base=base, device=devs[r])
        if b1 > b0:
            ix.append(slice_csr(corpus, b0, b1))
        g.attach_sparse(r, ix)
        parts.append(ix)
    return g, parts


def whole_index(corpus, bits=4, ub=1.0):
    n = len(corpus[0]) - 1
    ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=max(n, 1), capacity_pairs=len(corpus[1]) + 8)
    ix.append(corpus)
    return ix


def delete_everywhere(whole, parts, bounds, rows):
    rows = np.setdiff1d(np.asarray(rows, dtype=np.uint32), np.flatnonzero(whole.deleted_rows()[0])).astype(np.uint32)
    whole.delete_embedding(rows)
    for r, ix in enumerate(parts):
        mine = rows[(rows >= bounds[r]) & (rows < bounds[r + 1])] - bounds[r]
        if mine.size:
            ix.delete_embedding(mine)


def close(*xs):
    for x in xs:
        if isinstance(x, list):
            close(*x)
        else:
            x.close()


def launches(fn):
    before = cdb.kernel_launch_count()
    out = fn()
    return out, cdb.kernel_launch_count() - before


def quirky_corpus(seed, n_zipf):
    rows = quirky_rows(seed, 3000, 40)
    rows[5] = [(7, 0.0)]                        # touched only through zero products
    rows[6] = []                                # empty row: never a candidate
    rows[7] = [(3, 0.2), (3, 0.9), (3, 0.4)]    # duplicate dims
    return concat_csr([cdb.sparse_csr(rows), zipf_csr(seed + 1, n_zipf, vocab=40, mean_pairs=6)])


def quirky_queries(seed):
    queries = quirky_rows(seed, 40, 45)         # dims 40..44 are absent from the index
    queries[0] = []
    queries[1] = [(7, 0.0)]
    queries[2] = [(3, 0.5), (3, 0.5), (9, 2.0)]
    queries[3] = [(41, 1.0)]                    # no candidate anywhere
    return cdb.sparse_csr(queries)


@pytest.mark.parametrize("world,bits", [(2, 4), (3, 8), (4, 4), (4, 8)])
def test_group_equals_the_whole_index(world, bits):
    corpus = quirky_corpus(10 + world, 70_000)
    n = len(corpus[0]) - 1
    cuts = {2: [0, 9_000, n], 3: [0, 40_000, 41_500, n], 4: [0, 33_000, 34_000, 70_500, n]}[world]
    ub = 1.5 if bits == 8 else 1.0
    g, parts = sparse_group(corpus, cuts, bits, ub)
    whole = whole_index(corpus, bits, ub)
    q = quirky_queries(100 + world)
    for thr in THRS:
        for rerank in (False, True):
            same(g.search_sparse_all(q, opts_all(thr, rerank)), whole.batch_search_all(q, opts_all(thr, rerank)))
    got = g.search_sparse_all(q, opts_all(0.0, True))
    check_all(got, oracle_all(corpus, q, 0.0, True, bits, ub))
    assert got[0][4] == got[0][3]                                       # query 3: no candidate on any shard
    # deletes on every shard, the first results of some queries among them
    first = [int(got[1][got[0][i]]) for i in range(4, 10) if got[0][i + 1] > got[0][i]]
    delete_everywhere(whole, parts, cuts, np.concatenate([np.arange(3, n, 41), first, [cuts[1], cuts[-2]]]))
    deleted = whole.deleted_rows()[0]
    for thr, rerank in ((0.0, False), (0.0, True), (0.5, True), (float("nan"), False)):
        got = g.search_sparse_all(q, opts_all(thr, rerank))
        same(got, whole.batch_search_all(q, opts_all(thr, rerank)))
        assert not np.isin(got[1], np.flatnonzero(deleted)).any()
    check_all(g.search_sparse_all(q, opts_all(0.5, False)), oracle_all(corpus, q, 0.5, False, bits, ub, deleted))
    close(g, whole, parts)


def test_empty_and_all_deleted_shards_and_no_candidates():
    corpus = zipf_csr(31, 50_000, vocab=2000, mean_pairs=12)
    n = len(corpus[0]) - 1
    cuts = [0, 20_000, 20_000, 30_000, n]                  # shard 1 has no rows; shard 2's rows are all deleted below
    g, parts = sparse_group(corpus, cuts)
    whole = whole_index(corpus)
    delete_everywhere(whole, parts, cuts, np.arange(20_000, 30_000))
    q = concat_csr([zipf_csr(32, 30, vocab=2000, mean_pairs=6), cdb.sparse_csr([[], [(5000, 1.0)], [(1999, 0.0)]])])
    for rerank in (False, True):
        got = g.search_sparse_all(q, opts_all(0.0, rerank))
        same(got, whole.batch_search_all(q, opts_all(0.0, rerank)))
        assert not ((got[1] >= 20_000) & (got[1] < 30_000)).any()
        assert got[0][31] == got[0][30] and got[0][32] == got[0][31]   # an empty query, a dim no row has
    # every shard empty or fully deleted: no scoring, an empty handle
    delete_everywhere(whole, parts, cuts, np.arange(n))
    (off, ids, scores), k = launches(lambda: g.search_sparse_all(q, opts_all(0.0, True)))
    assert off.tolist() == [0] * 34 and len(ids) == 0 and len(scores) == 0 and k == 0
    close(g, whole, parts)


def test_skewed_corpus():
    """shard 1 owns almost every candidate: only its rows carry the queries' dims; the others touch a few"""
    a = zipf_csr(41, 30_000, vocab=500, mean_pairs=10)
    b = cdb.sparse_csr([[(d, 0.5 + (r % 7) * 0.25) for d in (600 + r % 3, 601)] for r in range(40_000)])
    c = zipf_csr(42, 20_000, vocab=500, mean_pairs=10)
    corpus = concat_csr([a, b, c])
    cuts = [0, 30_000, 70_000, 90_000]
    g, parts = sparse_group(corpus, cuts, bits=8, ub=2.0)
    whole = whole_index(corpus, bits=8, ub=2.0)
    q = cdb.sparse_csr([[(601, 1.0)], [(600, 0.3), (602, 2.0), (7, 0.1)], [(601, 0.2), (3, 1.0)]])
    for thr in (0.0, 0.5):
        for rerank in (False, True):
            same(g.search_sparse_all(q, opts_all(thr, rerank)), whole.batch_search_all(q, opts_all(thr, rerank)))
    off, ids, _ = g.search_sparse_all(q, opts_all(0.0))
    assert int(off[1]) == 40_000 and ((ids[:40_000] >= 30_000) & (ids[:40_000] < 70_000)).all()
    close(g, whole, parts)


def test_two_scoring_chunks_and_a_split_key_exchange():
    """four one-tile shards of 32768 rows that every query reaches through dim 0: a chunk is 511 queries, so 520 queries
    make two chunks, and a rank's 511 * 32768 keys exceed its share of the gather budget, so the first chunk's keys go in
    two sub-batches.  The plan is derived from the budget constants and the launches counted."""
    world, per = 4, 32768
    n = world * per
    rows = [[(0, 0.25 + (r % 13) * 0.125)] + ([(1 + r % 50, 1.0)] if r % 3 else []) for r in range(n)]
    corpus = cdb.sparse_csr(rows)
    cuts = [r * per for r in range(world + 1)]
    g, parts = sparse_group(corpus, cuts, bits=6, ub=2.0)
    whole = whole_index(corpus, bits=6, ub=2.0)
    nq = 520
    q = cdb.sparse_csr([[(0, 0.5 + (i % 5) * 0.3), (1 + i % 50, 0.7)] for i in range(nq)])
    counts = np.full((world, nq), per, np.int64)
    sizes, batches = sap.group_plan(counts, [(1, per)] * world)
    assert sizes == [511, 9] and len(batches[0]) >= 2
    for rerank in (False, True):
        got, k = launches(lambda: g.search_sparse_all(q, opts_all(0.0, rerank)))
        assert k == sap.group_launches(counts, [(1, per)] * world, rerank)
        assert np.array_equal(np.diff(got[0].astype(np.int64)), np.full(nq, n))
        same(got, whole.batch_search_all(q, opts_all(0.0, rerank)))
    sample = np.array([0, 255, 256, 510, 511, 519])
    check_all(got, oracle_all(corpus, sample_csr(q, sample), 0.0, True, 6, 2.0), sample)
    close(g, whole, parts)


def test_per_rank_group_of_one_equals_the_local_group():
    corpus = quirky_corpus(51, 40_000)
    ix = whole_index(corpus)
    ix.delete_embedding(np.arange(0, len(corpus[0]) - 1, 29, dtype=np.uint32))
    local = ShardGroup.local([0])
    local.attach_sparse(0, ix)
    rank = ShardGroup.rank(None, 1, 0, 0)
    rank.attach_sparse(0, ix)
    q = quirky_queries(52)
    for thr in (0.0, 1.0):
        for rerank in (False, True):
            want = ix.batch_search_all(q, opts_all(thr, rerank))
            same(rank.search_sparse_all(q, opts_all(thr, rerank)), want)
            same(local.search_sparse_all(q, opts_all(thr, rerank)), want)
    close(local, rank, ix)


def test_handle_is_independent_of_the_shards():
    L = _lib.load()
    corpus = zipf_csr(61, 60_000, vocab=1500, mean_pairs=15)
    cuts = [0, 25_000, 60_000]
    g, parts = sparse_group(corpus, cuts, room=5000)
    q = zipf_csr(62, 20, vocab=1500, mean_pairs=6)
    o, d, v = q
    p = opts_all(0.0, True).params()
    h = C.c_void_p()
    assert L.cdb_sparse_search_batch_all_sharded(g._h, o.ctypes.data, d.ctypes.data, v.ctypes.data, len(o) - 1, C.byref(p),
                                                 C.byref(h)) == 0
    r = SparseResults(h)
    off = r.offsets()
    full = r.read(0, len(off) - 1)
    same((off,) + full, g.search_sparse_all(q, opts_all(0.0, True)))
    parts[1].append(zipf_csr(63, 3000, vocab=1500, mean_pairs=15))
    parts[0].delete_embedding(full[0][full[0] < 25_000][:40])
    assert not np.array_equal(g.search_sparse_all(q, opts_all(0.0, True))[1], full[0])
    g.close()
    close(parts)
    assert np.array_equal(r.offsets(), off)
    got = r.read(0, len(off) - 1)
    assert np.array_equal(got[0], full[0]) and np.array_equal(got[1].view(np.uint32), full[1].view(np.uint32))
    r.close()


def test_refusals_and_the_empty_batch():
    L = _lib.load()
    inv = cdb.Status.INVALID_PARAMS
    err = lambda: (L.cdb_last_error_string() or b"").decode()   # noqa: E731
    corpus = zipf_csr(71, 1000, vocab=100, mean_pairs=5)
    g, parts = sparse_group(corpus, [0, 400, 1000])
    qo, qd, qv = np.array([0, 1], np.uint64), np.array([1], np.uint32), np.array([1.0], np.float32)
    out = C.c_void_p(1)

    def call(grp, p, o=qo, nq=1, d=qd, v=qv):
        return L.cdb_sparse_search_batch_all_sharded(grp, o.ctypes.data if o is not None else None, d.ctypes.data if d is not None else None,
                                                     v.ctypes.data, nq, C.byref(p), C.byref(out))

    assert call(g._h, cdb.SparseSearchOptions(10).params()) == inv and "k = 0" in err()
    assert out.value is None
    assert call(g._h, opts_all().params(), o=np.array([0, 2, 1], np.uint64), nq=2) == inv and "offsets decrease" in err()
    assert call(g._h, opts_all().params(), d=None) == inv and "null query pairs" in err()
    with pytest.raises(cdb.CosdataError) as e:
        g.search_sparse_all([[(1, 1.0)]], cdb.SparseSearchOptions(5))
    assert e.value.status == inv
    # a slot without a sparse shard, refused before any device work
    half = ShardGroup.local(devices(2))
    half.attach_sparse(0, parts[0])
    before = cdb.kernel_launch_count()
    assert call(half._h, opts_all().params()) == inv and "no sparse shard" in err()
    assert cdb.kernel_launch_count() == before
    # n_queries = 0: a handle of 0 queries, nothing launched
    (off, ids, _), k = launches(lambda: g.search_sparse_all([], opts_all(0.0, True)))
    assert off.tolist() == [0] and len(ids) == 0 and k == 0
    close(g, half, parts)
